// Masked-window attention on Hopper tensor cores (SparseWindowAttention, sparse_transformer.py:327-357).
//
// One CTA (256 threads = two warpgroups, two CTAs per SM) per (128-query tile, 5x9 window, head, sliding window);
// warpgroup w owns query rows 64w..64w+63.  Per 64-key tile:
//   S = Q K^T       wgmma m64n64k16 x8 (K = 128 = d)                    -> registers
//   softmax         in registers: a query row lives on the 4 threads of a quad (row max / sum by two shuffles),
//                   P (fp16) written to shared memory as the next A operand
//   O += P V        wgmma m64n128k16 x4 (K = 64 keys), V as the MN-major B operand  -> registers
// The running max is only raised when it grew by more than 8 (log2 units), in which case the O rows are rescaled;
// softmax is invariant to that shift, so the result is exact while P stays within fp16 range (<= 2^8).
// Keys are gathered by index (own 45 + ring 148 + pooled tokens of every 2nd frame) with 16-byte cp.async into
// 128B-swizzled panels -- the window/rolled/pooled K,V tensors of the reference are never materialised.
#include "attention.cuh"
#include "wgmma_ops.cuh"

namespace {

constexpr int D = 128, BQ = 128, BKEY = 64, NT = 256, WIN_TOK = 45, RING = 193;
constexpr uint32_t QPANEL = BQ * 128;           // bytes of a [128 rows][64 halves] panel (Q, P)
constexpr uint32_t KPANEL = BKEY * 128;         // bytes of a [BKEY rows][64 halves] panel (K, V)
constexpr uint32_t QTILE = 2 * QPANEL;          // Q: [128][128 d]
constexpr uint32_t KTILE = 2 * KPANEL;          // K or V: [BKEY][128 d]
constexpr uint32_t PTILE = (BKEY / 64) * QPANEL;  // P: [128][BKEY keys]
// 112 KiB per CTA so that two CTAs share an SM: one CTA's softmax overlaps the other's MMAs and gathers
constexpr uint32_t SM_Q = 0, SM_K = QTILE, SM_V = SM_K + 2 * KTILE, SM_P = SM_V + 2 * KTILE, SM_END = SM_P + PTILE;

// byte offset of 16-byte chunk `chunk` (along the 64-wide panels) of row `row` in a tile whose panels are `panel` bytes
__device__ __forceinline__ uint32_t tile_off(uint32_t panel, int row, int chunk) {
  return (uint32_t)(chunk >> 3) * panel + (uint32_t)row * 128 + (uint32_t)(((chunk & 7) ^ (row & 7)) << 4);
}

// Key-row gather table: entry j of window `win` is the source row of key j of a masked window, as an offset (in
// 16-byte units, relative to the first frame of the sliding window) into the K/V token tensor, or -- top bit set --
// into the pooled K/V tensor.  Keys of T_ind frame fi (frame parity + 2*fi) are [own 45 | ring 148 | pooled n_pool].
// Built once per launch so that the gather loop of the attention kernel does no integer division or index math.
__global__ void attn_key_table(int* __restrict__ tab, const int* __restrict__ ring_idx, int nk_max, int kpf, int ntok,
                               int n_pool, int qkv_cs, int pool_cs, int parity) {
  const int win = blockIdx.x;
  const int* ring = ring_idx + win * RING;
  for (int j = threadIdx.x; j < nk_max; j += blockDim.x) {
    const int fi = j / kpf, w = j - fi * kpf;
    const int fr = parity + 2 * fi;
    unsigned e;
    if (w < RING) e = (unsigned)(((long long)fr * ntok + ring[w]) * qkv_cs / 8);
    else e = 0x80000000u | (unsigned)(((long long)fr * n_pool + (w - RING)) * pool_cs / 8);
    tab[(long long)win * nk_max + j] = (int)e;
  }
}

__global__ void __launch_bounds__(NT, 2) window_attention_tc(const PPAttnParams p) {
  using namespace ppx;
  extern __shared__ __align__(1024) uint8_t smem[];   // 128B-swizzled tiles need 1024-byte alignment
  const uint32_t sbase = smem_u32(smem);

  const int win = blockIdx.y >> 2, head = blockIdx.y & 3, sw = blockIdx.z;
  if (p.win_flags[sw * p.n_win + win] == 0) return;        // unmasked windows: mma.sync kernel
  const int t = p.sw_t[sw];
  const int frame_base = p.sw_frame_off[sw];
  const int nq = t * WIN_TOK;
  const int q0 = blockIdx.x * BQ;
  if (q0 >= nq) return;
  const int n_tind = (t - p.parity + 1) / 2;
  const int kpf = RING + p.n_pool;
  const int nk = n_tind * kpf;
  const int ntiles = (nk + BKEY - 1) / BKEY;
  const int tid = threadIdx.x;
  const int* ring = p.ring_idx + win * RING;
  const long long ntok = (long long)p.nh * p.nw;

  // ---- Q tile (rows beyond nq are clamped to a valid query; never stored)
  for (int i = tid; i < BQ * 16; i += NT) {
    const int r = i >> 4, ch = i & 15;
    const int qi = min(q0 + r, nq - 1);
    const int fr = frame_base + qi / WIN_TOK, pos = qi % WIN_TOK;
    const __half* src = p.q + ((long long)fr * ntok + ring[pos]) * p.qkv_cs + head * D + ch * 8;
    cp_async16(sbase + SM_Q + tile_off(QPANEL, r, ch), src, 16);
  }
  // K/V gather: thread owns 16-byte chunk `ch` of rows r0, r0+16, r0+32, r0+48 of every key tile; the source row of
  // key j comes from the per-window table (attn_key_table), so the loop body is a table load, two adds and two copies
  const int r0 = tid >> 4, ch = tid & 15;
  const long long fb = frame_base;
  const __half* kb = p.k + fb * ntok * p.qkv_cs + head * D + ch * 8;
  const __half* vb = p.v + fb * ntok * p.qkv_cs + head * D + ch * 8;
  const __half* pkb = p.pk + fb * p.n_pool * p.pool_cs + head * D + ch * 8;
  const __half* pvb = p.pv + fb * p.n_pool * p.pool_cs + head * D + ch * 8;
  const int* ktab = p.key_tab + (long long)win * p.key_tab_stride;
  const uint32_t kv_dst0 = sbase + tile_off(KPANEL, r0, ch);
  auto load_kv = [&](int tile, int stage) {
    const uint32_t dk = kv_dst0 + SM_K + stage * KTILE, dv = kv_dst0 + SM_V + stage * KTILE;
#pragma unroll
    for (int it = 0; it < BKEY / 16; ++it) {
      const int j = tile * BKEY + r0 + 16 * it;
      const __half* ks = kb; const __half* vs = vb;
      uint32_t nbytes = 0;
      if (j < nk) {
        nbytes = 16;
        const int e = __ldg(ktab + j);
        const long long off = (long long)(e & 0x7fffffff) * 8;
        ks = (e < 0 ? pkb : kb) + off;
        vs = (e < 0 ? pvb : vb) + off;
      }
      cp_async16(dk + it * 2048, ks, nbytes);     // rows r0 + 16*it: same swizzle phase, 16 rows * 128 B further
      cp_async16(dv + it * 2048, vs, nbytes);
    }
    cp_async_commit();
  };
  load_kv(0, 0);   // one group: Q + first K/V tile

  // fragment coordinates (pp_common.cuh): this thread holds rows rw and rw + 8 of its warpgroup's 64, and per 8-column
  // group the two columns 2 * quad .. +1
  const int wg = tid >> 7, lane = tid & 31;
  const int rw = 16 * ((tid >> 5) & 3) + (lane >> 2), quad = lane & 3;
  const uint32_t q_rows = (uint32_t)wg * 64 * 128;   // byte offset of this warpgroup's rows in a [128][64] panel
  float o[64];
  float m_used[2] = {0.f, 0.f}, m_run[2] = {-1e30f, -1e30f}, row_sum[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  for (int j = 0; j < ntiles; ++j) {
    const int stage = j & 1;
    cp_async_wait<0>();
    fence_proxy_async();
    __syncthreads();   // K/V tile j has landed; both warpgroups are done with tile j-1 (its stage is free again)
    if (j + 1 < ntiles) load_kv(j + 1, stage ^ 1);
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t sub = (uint32_t)(ks & 3) * 32;
      wgmma_f16<BKEY>(s, gmma_desc_sw128_kmajor(sbase + SM_Q + (uint32_t)(ks >> 2) * QPANEL + q_rows + sub),
                      gmma_desc_sw128_kmajor(sbase + SM_K + stage * KTILE + (uint32_t)(ks >> 2) * KPANEL + sub), ks != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);

    const int kvalid = min(BKEY, nk - j * BKEY);
    float mx[2] = {-1e30f, -1e30f};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (8 * (i >> 2) + 2 * quad + (i & 1) >= kvalid) s[i] = -1e30f;
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    }
    float f[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      // the reference max is kept in fp16 precision; any reference works for softmax as long as numerator and
      // denominator share it
      const float m_tile = __half2float(__float2half_rn(fmaxf(mx[h] * p.scale_log2, -60000.f)));
      const float m_new = fmaxf(m_run[h], m_tile);
      f[h] = 1.f;
      if (j == 0) m_used[h] = m_new;
      else if (m_new > m_used[h] + 8.f) {   // rare: raise the reference max and rescale the row
        f[h] = exp2f(m_used[h] - m_new);
        m_used[h] = m_new;
        row_sum[h] *= f[h];
      }
      m_run[h] = m_new;
    }
    if (f[0] != 1.f || f[1] != 1.f) {
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] *= f[(i >> 1) & 1];
    }
    // ---- P = exp2(s*scale - m_used) -> shared memory (A operand of P.V)
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const float a = exp2f(fmaf(s[i], p.scale_log2, -m_used[h]));
      const float b = exp2f(fmaf(s[i + 1], p.scale_log2, -m_used[h]));
      row_sum[h] += a + b;
      const int row = wg * 64 + rw + 8 * h;
      *reinterpret_cast<__half2*>(smem + SM_P + tile_off(QPANEL, row, i >> 2) + 4 * quad) = __floats2half2_rn(a, b);
    }
    fence_proxy_async();
    named_bar(1 + wg, 128);   // this warpgroup's P rows are complete
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BKEY / 16; ++ks) {
      const uint64_t adesc = gmma_desc_sw128_kmajor(sbase + SM_P + q_rows + (uint32_t)ks * 32);
      const uint64_t bdesc = gmma_desc_sw128_mnmajor(sbase + SM_V + stage * KTILE + (uint32_t)ks * 2048, KPANEL);
      wgmma_f16<D, 1>(o, adesc, bdesc, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
  }

  // ---- epilogue: O / row_sum -> global (unpadded grid; padding queries are dropped)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row_sum[h] += __shfl_xor_sync(0xffffffffu, row_sum[h], 1);
    row_sum[h] += __shfl_xor_sync(0xffffffffu, row_sum[h], 2);
    const float inv = 1.f / row_sum[h];
    const int qi = q0 + wg * 64 + rw + 8 * h;
    if (qi >= nq) continue;
    const int fr = frame_base + qi / WIN_TOK, pos = qi % WIN_TOK;
    const int tok = ring[pos];
    const int ty = tok / p.nw, tx = tok - ty * p.nw;
    if (ty >= p.gh || tx >= p.gw) continue;
    __half* dst = p.out + (((long long)fr * p.gh + ty) * p.gw + tx) * p.out_cs + head * D + 2 * quad;
#pragma unroll
    for (int g = 0; g < D / 8; ++g)
      *reinterpret_cast<__half2*>(dst + 8 * g) = __floats2half2_rn(o[4 * g + 2 * h] * inv, o[4 * g + 2 * h + 1] * inv);
  }
}

}  // namespace

int pp_launch_attention_tc(const PPAttnParams& p, int n_sliding, int t_max, cudaStream_t st) {
  const size_t smem = SM_END;   // 112 KiB: two CTAs per SM
  static bool attr_set = false;
  if (!attr_set) {
    PP_CUDA_CHECK(cudaFuncSetAttribute(window_attention_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PP_CUDA_CHECK(cudaFuncSetAttribute(window_attention_tc, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    attr_set = true;
  }
  {
    const int kpf = RING + p.n_pool, nk_max = ((t_max - p.parity + 1) / 2) * kpf;
    PP_REQUIRE(p.key_tab != nullptr && p.key_tab_stride >= nk_max, "attention: key table scratch too small (%d < %d)",
               p.key_tab_stride, nk_max);
    attn_key_table<<<p.n_win, 256, 0, st>>>(const_cast<int*>(p.key_tab), p.ring_idx, p.key_tab_stride, kpf, p.nh * p.nw, p.n_pool,
                                           p.qkv_cs, p.pool_cs, p.parity);
    PP_CUDA_CHECK(cudaGetLastError());
  }
  dim3 grid(pp_ceil_div(t_max * WIN_TOK, BQ), p.n_win * 4, n_sliding);
  window_attention_tc<<<grid, NT, smem, st>>>(p);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

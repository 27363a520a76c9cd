// Stage 1: bidirectional RAFT optical flow (reference: model/modules/flow_comp_raft.py:39-58,
// model/modules/RAFT/raft.py:94-152).  Result-identical restructuring vs the reference:
//   * fnet / cnet run once per frame (InstanceNorm is per-sample, BatchNorm is in eval mode), not once per
//     pair and direction;
//   * all pairs of both directions are batched (pairs are independent), bounded only by workspace;
//   * the mask head and convex upsampling run only after the last GRU iteration (raft.py:141-150 keeps
//     only the last flow_up).
// Two precisions share this code.  fp16: fp16 activations and correlation pyramid, fp32 accumulation.  fp32 (the node's
// fp16="disable"): every activation is an fp32 split-tf32 pair tensor [pix][hi C | lo C] and every convolution and the
// correlation GEMM run as 3xTF32 (conv_igemm.cuh), the pyramid is fp32; only the accumulation order differs from fp32.
#include <string.h>

#include "engine.cuh"

namespace {

// An activation tensor of the stage's precision: fp16 [pix][C], or (fp32) a split pair tensor float [pix][hi C | lo C].
struct Act {
  void* p;
  int C;
  __half* h() const { return reinterpret_cast<__half*>(p); }
  float* f() const { return reinterpret_cast<float*>(p); }
};

int alloc_act(PPEngine& e, bool fp32, Act& a, long long pixels, int C, const char* what) {
  uint8_t* ptr = nullptr;
  PP_TRY(pp_alloc(e, &ptr, (size_t)pixels * C * (fp32 ? 8 : 2), what));
  a = Act{ptr, C};
  return PP_OK;
}

// One convolution in the stage's precision (fp32: the layer's split weight image "<name>.tf32").  Channel offsets and
// counts are real channels in both precisions.
struct RConv {
  PPConvCall c;
  bool f32;
  RConv(PPEngine& e, bool fp32, const std::string& name, int N, int H, int W)
      : c(e, fp32 ? name + ".tf32" : name, N, H, W), f32(fp32) {
    if (f32) c.tf32();
  }
  RConv& in(const Act& t, int co, int channels) {
    if (f32) c.in_split(t.f(), t.C, co, channels);
    else c.in(t.h(), t.C, co, channels);
    return *this;
  }
  RConv& geom(int sh, int sw, int ph, int pw) { c.geom(sh, sw, ph, pw); return *this; }
  RConv& out(const Act& t, int co) {
    if (f32) c.out_split(t.f(), t.C, co);
    else c.out(t.p, t.C, co);
    return *this;
  }
  RConv& out_plain_f32(float* ptr, int cs) { c.out(ptr, cs, 0, 1); return *this; }
  RConv& act(int act1, float slope = 0.f, float scale = 1.f, int act2 = PP_ACT_NONE) {
    c.act(act1, slope, scale, act2);
    return *this;
  }
  RConv& residual(const Act& t, int co) {
    if (f32) c.residual_split(t.f(), t.C, co);
    else c.residual(t.h(), t.C, co);
    return *this;
  }
  RConv& gru_zr(const Act& h, int h_co, const Act& rh, int rh_co) {
    if (f32) c.gru_zr_split(h.f(), h.C, h_co, rh.f(), rh.C, rh_co);
    else c.gru_zr(h.h(), h.C, h_co, rh.h(), rh.C, rh_co);
    return *this;
  }
  RConv& gru_h(const Act& h, int h_co, const Act& z, int z_co) {
    if (f32) c.gru_h_split(h.f(), h.C, h_co, z.f(), z.C, z_co);
    else c.gru_h(h.h(), h.C, h_co, z.h(), z.C, z_co);
    return *this;
  }
  int run(cudaStream_t st) { return c.run(st); }
};

struct Enc {
  PPEngine& e;
  cudaStream_t st;
  std::string pre;  // "raft.fnet." / "raft.cnet."
  bool inst;
  float* sums;      // [n][2][C] scratch for instance norm
  bool f32;
};

// conv (+ instance norm or folded batch norm) (+ relu) (+ residual, relu)
int enc_conv(Enc& c, const std::string& name, const Act& x, int n, int H, int W, int stride, const Act& out, bool relu,
             const Act* residual) {
  RConv call(c.e, c.f32, c.pre + name, n, H, W);
  call.in(x, 0, x.C);
  const int kh = call.c.p.kh, kw = call.c.p.kw;
  call.geom(stride, stride, (kh - 1) / 2, (kw - 1) / 2);
  const int OH = (H + 2 * ((kh - 1) / 2) - (kh - 1) - 1) / stride + 1;
  const int OW = (W + 2 * ((kw - 1) / 2) - (kw - 1) - 1) / stride + 1;
  if (c.inst) {
    // raw conv output -> statistics -> normalise in place (+relu, +residual)
    call.out(out, 0);
    PP_TRY(call.run(c.st));
    if (c.f32) {
      PP_TRY(pp_k_instnorm_stats_f32(out.f(), n, OH * OW, out.C, c.sums, c.st));
      PP_TRY(pp_k_instnorm_apply_f32(out.f(), c.sums, residual ? residual->f() : nullptr, out.f(), n, OH * OW, out.C,
                                     relu ? 1 : 0, c.st));
    } else {
      PP_TRY(pp_k_instnorm_stats(out.h(), n, OH * OW, out.C, c.sums, c.st));
      PP_TRY(pp_k_instnorm_apply(out.h(), c.sums, residual ? residual->h() : nullptr, out.h(), n, OH * OW, out.C,
                                 relu ? 1 : 0, c.st));
    }
    c.e.launches += c.f32 ? 5 : 3;  // memset + 2 kernels (fp32: the statistics take two passes)
  } else {
    call.out(out, 0);
    if (residual != nullptr) call.act(relu ? PP_ACT_RELU : PP_ACT_NONE, 0.f, 1.f, PP_ACT_RELU).residual(*residual, 0);
    else call.act(relu ? PP_ACT_RELU : PP_ACT_NONE);
    PP_TRY(call.run(c.st));
  }
  return PP_OK;
}

// BasicEncoder on n frames: x [n][H][W][x.C] -> out [n][H/8][W/8][256]
int encoder(Enc& c, const Act& x, int n, int H, int W, const Act& out) {
  PPEngine& e = c.e;
  const size_t mark = e.arena.mark();
  const int h2 = (H + 2 * 3 - 7) / 2 + 1, w2 = (W + 2 * 3 - 7) / 2 + 1;
  const long long px = (long long)n * h2 * w2;
  Act a, b, y;
  PP_TRY(alloc_act(e, c.f32, a, px, 64, "raft enc a"));
  PP_TRY(alloc_act(e, c.f32, b, px, 64, "raft enc b"));
  PP_TRY(alloc_act(e, c.f32, y, px, 64, "raft enc y"));
  PP_TRY(enc_conv(c, "conv1", x, n, H, W, 2, a, true, nullptr));
  Act cur = a, nxt = b;
  int hh = h2, ww = w2;
  const int dims[3] = {64, 96, 128};
  for (int li = 0; li < 3; ++li) {
    for (int bi = 0; bi < 2; ++bi) {
      const int s = (li > 0 && bi == 0) ? 2 : 1;
      const int co = dims[li];
      const std::string q = "layer" + std::to_string(li + 1) + "." + std::to_string(bi) + ".";
      const int oh = (hh + 2 - 3) / s + 1, ow = (ww + 2 - 3) / s + 1;
      // the buffers hold 64 channels at h2 x w2: every later layer has at most as many values per image
      Act y1{y.p, co}, nx{nxt.p, co}, cu{cur.p, co};
      // y1 = relu(norm1(conv1(x)))
      PP_TRY(enc_conv(c, q + "conv1", cur, n, hh, ww, s, y1, true, nullptr));
      if (s != 1) {
        // x = norm3(downsample(x)) -- written into nxt first, then used as the residual of conv2 in place
        PP_TRY(enc_conv(c, q + "downsample", cur, n, hh, ww, s, nx, false, nullptr));
        // out = relu(x + relu(norm2(conv2(y1)))) -> needs a third buffer: reuse `cur` (its content is dead now)
        PP_TRY(enc_conv(c, q + "conv2", y1, n, oh, ow, 1, cu, true, &nx));
        cur = cu;   // result is in cur
      } else {
        PP_TRY(enc_conv(c, q + "conv2", y1, n, oh, ow, 1, nx, true, &cur));
        nxt = cur;
        cur = nx;
      }
      hh = oh; ww = ow;
    }
  }
  PP_TRY(RConv(e, c.f32, c.pre + "conv2", n, hh, ww).in(cur, 0, cur.C).geom(1, 1, 0, 0).out(out, 0).run(c.st));
  e.arena.release(mark);
  return PP_OK;
}

}  // namespace

int pp_raft_corr_pad(int P) {
  const int ntile = pp_ceil_div(P, 256);
  return ((pp_ceil_div(P, ntile) + 15) / 16) * 16 * ntile;
}

int pp_raft_corr_volume(PPEngine& e, const void* fmap1, const void* fpack2, int pairs, int P, int P_pad, bool fp32,
                        void* corr0, cudaStream_t st) {
  // all-pairs correlation: grouped GEMM, one group per frame pair, scaled by 1/sqrt(256)
  PP_REQUIRE((long long)P * P < (1LL << 31), "raft: frame too large for the correlation volume indexing");
  const size_t cb = fp32 ? 4 : 2;
  const int fk = fp32 ? 3 * 256 : 256;
  const long long Ms = (long long)pairs * P;
  PPConvParams p;
  memset(&p, 0, sizeof(p));
  if (fp32) {
    // A = fmap1 read as (hi, lo, hi), in the kernel's 2-byte units (conv_igemm.cuh); B = the [hi; hi; lo] image
    PP_REQUIRE((long long)pairs * P * 1024 < (1LL << 31), "raft: too many frame pairs for one correlation launch");
    p.split = 1;
    p.nseg = 3;
    for (int k = 0; k < 3; ++k) {
      p.seg[k].ptr = reinterpret_cast<const __half*>(fmap1);
      p.seg[k].cstride = 1024; p.seg[k].coff = k == 1 ? 512 : 0;
      p.seg[k].gstep = P * 1024; p.seg[k].cbegin = 512 * k; p.seg[k].cend = 512 * (k + 1);
    }
    p.Cin = 1536;
  } else {
    p.nseg = 1;
    p.seg[0].ptr = reinterpret_cast<const __half*>(fmap1); p.seg[0].cstride = 256; p.seg[0].coff = 0;
    p.seg[0].gstep = P * 256; p.seg[0].cbegin = 0; p.seg[0].cend = 256;
    p.Cin = 256;
  }
  p.wpacked = reinterpret_cast<const __half*>(fpack2);
  p.N = 1; p.H = 1; p.W = P; p.OH = 1; p.OW = P;
  p.kh = p.kw = 1; p.sh = p.sw = 1; p.dh = p.dw = 1;
  p.bias = nullptr;
  p.Cout_g = P; p.Cout_g_pad = P_pad; p.BN = P_pad / pp_ceil_div(P, 256); p.groups = pairs;
  p.epi = PP_EPI_STD; p.scale = 1.f / 16.f;
  // group g writes rows [g*P, (g+1)*P): out index = m*out_cstride + out_coff + g*out_gstep + n
  // (P*P exceeds the int range only beyond 46340 pixels at 1/8 res, i.e. 3.7 MPixel frames)
  p.out = corr0; p.out_cstride = P; p.out_coff = 0; p.out_fp32 = fp32 ? 1 : 0;
  p.out_gstep = P * P;
  {
    PPProfScope ps(e, "conv:igemm:raft.corr", (double)Ms, 2.0 * Ms * P * fk, (double)Ms * P * cb + 2.0 * Ms * fk * cb, st);
    PP_TRY(pp_launch_conv(p, st));
  }
  e.launches++;
  return PP_OK;
}

int pp_raft_corr_pool(PPEngine& e, void* const corr[4], long long M, int h8, int w8, bool fp32, cudaStream_t st) {
  for (int l = 0; l < 3; ++l) {
    const int h = h8 >> l, w = w8 >> l;
    if (fp32) PP_TRY(pp_k_corr_pool_f32(static_cast<float*>(corr[l]), static_cast<float*>(corr[l + 1]), M, h, w, st));
    else PP_TRY(pp_k_corr_pool(static_cast<__half*>(corr[l]), static_cast<__half*>(corr[l + 1]), M, h, w, st));
    e.launches++;
  }
  return PP_OK;
}

int pp_stage_raft(PPEngine& e, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                  bool fp32, cudaStream_t st) {
  PP_REQUIRE(T >= 2, "raft: need at least 2 frames, got %d", T);
  PP_REQUIRE(H % 8 == 0 && W % 8 == 0, "raft: size %dx%d must be a multiple of 8", W, H);
  PP_REQUIRE((H / 8) >= 16 && (W / 8) >= 16, "raft: H/8 and W/8 must be >= 16 (4-level correlation pyramid)");
  const int h8 = H / 8, w8 = W / 8, P = h8 * w8;
  const size_t mark0 = e.arena.mark();
  const size_t cb = fp32 ? 4 : 2;        // bytes per correlation value / per packed fmap value
  const int fk = fp32 ? 3 * 256 : 256;   // K of the correlation GEMM (fp32: the segments (hi, lo, hi))

  // ---- per-frame encoders ------------------------------------------------------------------------
  Act fmap, cmap;
  uint8_t* fpack;
  int P_pad;
  P_pad = pp_raft_corr_pad(P);
  PP_TRY(alloc_act(e, fp32, fmap, (long long)T * P, 256, "fmap"));
  PP_TRY(alloc_act(e, fp32, cmap, (long long)T * P, 256, "cmap"));
  PP_TRY(pp_alloc(e, &fpack, (size_t)T * P_pad * fk * cb, "fmap packed"));
  {
    const size_t m1 = e.arena.mark();
    const long long half_px = (long long)(H / 2) * (W / 2);
    int chunk = (int)((8LL << 20) / half_px);
    if (chunk < 1) chunk = 1;
    if (chunk > T) chunk = T;
    Act x;                               // fp16: 3 + 5 zero channels; fp32: 3 + 1 zero channel (16-byte vectors)
    float* sums;
    PP_TRY(alloc_act(e, fp32, x, (long long)chunk * H * W, fp32 ? 4 : 8, "raft input"));
    PP_TRY(pp_alloc(e, &sums, pp_k_instnorm_scratch_floats(chunk, (H / 2) * (W / 2), 256), "instnorm sums"));
    const size_t fbytes = (size_t)P * 256 * (fp32 ? 8 : 2);   // one frame of fmap / cmap
    for (int f0 = 0; f0 < T; f0 += chunk) {
      const int n = (f0 + chunk <= T) ? chunk : T - f0;
      if (fp32) PP_TRY(pp_k_nchw_f32_to_split(frames + (size_t)f0 * 3 * H * W, x.f(), n, 3, H, W, 4, st));
      else PP_TRY(pp_k_nchw_f32_to_nhwc_f16(frames + (size_t)f0 * 3 * H * W, x.h(), n, 3, H, W, 8, 0, 8, st));
      e.launches++;
      Enc fe{e, st, "raft.fnet.", true, sums, fp32};
      PP_TRY(encoder(fe, x, n, H, W, Act{(uint8_t*)fmap.p + f0 * fbytes, 256}));
      Enc ce{e, st, "raft.cnet.", false, sums, fp32};
      PP_TRY(encoder(ce, x, n, H, W, Act{(uint8_t*)cmap.p + f0 * fbytes, 256}));
    }
    e.arena.release(m1);
  }
  if (fp32) PP_TRY(pp_k_pack_b_operand_split(fmap.f(), reinterpret_cast<float*>(fpack), T, P, P_pad, 256, st));
  else PP_TRY(pp_k_pack_b_operand(fmap.h(), reinterpret_cast<__half*>(fpack), T, P, P_pad, 256, st));
  e.launches++;

  // ---- pair batches -----------------------------------------------------------------------------
  const int lvl_h[4] = {h8, h8 >> 1, h8 >> 2, h8 >> 3}, lvl_w[4] = {w8, w8 >> 1, w8 >> 2, w8 >> 3};
  size_t corr_elems = 0;
  for (int l = 0; l < 4; ++l) corr_elems += (size_t)P * lvl_h[l] * lvl_w[l];
  // lookup output: 324 channels padded to 328 (fp16) / 352 (fp32: 32-channel K chunks of the split segments)
  const int lk_C = fp32 ? 352 : 328;
  // per pair: pyramid, activations (hx rh z lk c1 corflo f1 patches fh, fp16: + flow8), coords + delta, slack, mask
  const size_t per_pair = fp32 ? corr_elems * 4 + (size_t)P * (384 + 128 + 128 + lk_C + 256 + 256 + 128 + 128 + 256) * 8 +
                                     (size_t)P * 4 * 4 + (size_t)P * 32 * 4 + (size_t)P * 576 * 8
                               : corr_elems * 2 + (size_t)P * (384 + 128 + 128 + 328 + 256 + 256 + 128 + 128 + 8 + 256) * 2 +
                                     (size_t)P * 4 * 4 + (size_t)P * 32 * 4 + (size_t)P * 576 * 2;
  const size_t avail = e.arena.cap - e.arena.off;
  int max_pairs = (int)(avail * 9 / 10 / per_pair);
  PP_REQUIRE(max_pairs >= 1, "raft: workspace too small for one frame pair (%zu bytes needed)", per_pair);
  const int npairs = T - 1;

  // Both directions share one batch: pair slot s < npairs is the forward pair (s -> s+1), slot npairs + s the backward
  // pair (s+1 -> s).  One launch per layer then covers 2(T-1) pairs (half as many launches and tile-quantisation
  // tails on the SMs as one batch per direction); only the steps that address frames (correlation, context
  // split, final upsampling) run once per direction sub-range of the batch.
  struct Sub { int dir, b0, cnt, off; };   // direction, first pair of that direction, count, slot offset in the batch
  for (int s0 = 0; s0 < 2 * npairs; s0 += max_pairs) {
    {
      const int B = (s0 + max_pairs <= 2 * npairs) ? max_pairs : 2 * npairs - s0;
      Sub subs[2];
      int nsub = 0;
      for (int d = 0; d < 2; ++d) {
        const int lo = s0 > d * npairs ? s0 : d * npairs;
        const int hi = (s0 + B) < (d + 1) * npairs ? (s0 + B) : (d + 1) * npairs;
        if (hi > lo) subs[nsub++] = Sub{d, lo - d * npairs, hi - lo, lo - s0};
      }
      const size_t m2 = e.arena.mark();
      const long long M = (long long)B * P;
      void* corr[4];
      for (int l = 0; l < 4; ++l) {
        uint8_t* c;
        PP_TRY(pp_alloc(e, &c, (size_t)M * lvl_h[l] * lvl_w[l] * cb, "corr level"));
        corr[l] = c;
      }
      for (int si = 0; si < nsub; ++si) {
        const Sub& sb = subs[si];
        const int f1 = sb.dir == 0 ? sb.b0 : sb.b0 + 1;  // first frame playing image1
        const int f2 = sb.dir == 0 ? sb.b0 + 1 : sb.b0;  // first frame playing image2
        PP_TRY(pp_raft_corr_volume(e, (const uint8_t*)fmap.p + (size_t)f1 * P * 256 * (fp32 ? 8 : 2),
                                   fpack + (size_t)f2 * P_pad * fk * cb, sb.cnt, P, P_pad, fp32,
                                   static_cast<uint8_t*>(corr[0]) + (size_t)sb.off * P * P * cb, st));
      }
      PP_TRY(pp_raft_corr_pool(e, corr, M, h8, w8, fp32, st));
      // GRU state and scratch
      Act hx, rh, z, lk, c1, corflo, f1b, fpatch, fh;
      __half* flow8 = nullptr;                 // fp16 only: the flow for the 7x7 patches (fp32 takes it from coords1)
      float *coords1, *delta;
      PP_TRY(alloc_act(e, fp32, hx, M, 384, "hx"));
      PP_TRY(alloc_act(e, fp32, rh, M, 128, "rh"));
      PP_TRY(alloc_act(e, fp32, z, M, 128, "z"));
      PP_TRY(alloc_act(e, fp32, lk, M, lk_C, "corr lookup"));
      PP_TRY(alloc_act(e, fp32, c1, M, 256, "c1"));
      PP_TRY(alloc_act(e, fp32, corflo, M, 256, "corflo"));
      PP_TRY(alloc_act(e, fp32, f1b, M, 128, "f1"));
      PP_TRY(alloc_act(e, fp32, fpatch, M, 128, "flow patches"));
      if (!fp32) PP_TRY(pp_alloc(e, &flow8, (size_t)M * 8, "flow8"));
      PP_TRY(alloc_act(e, fp32, fh, M, 256, "flow head"));
      PP_TRY(pp_alloc(e, &coords1, (size_t)M * 2, "coords1"));
      PP_TRY(pp_alloc(e, &delta, (size_t)M * 2, "delta"));
      for (int si = 0; si < nsub; ++si) {
        const int f1 = subs[si].dir == 0 ? subs[si].b0 : subs[si].b0 + 1;
        const long long npx = (long long)subs[si].cnt * P;
        if (fp32)
          PP_TRY(pp_k_cnet_split_f32(cmap.f() + (size_t)f1 * P * 512, hx.f() + (size_t)subs[si].off * P * 768, 384, npx, st));
        else
          PP_TRY(pp_k_cnet_split(cmap.h() + (size_t)f1 * P * 256, hx.h() + (size_t)subs[si].off * P * 384, 384, npx, st));
        e.launches++;
      }
      if (fp32) PP_TRY(pp_k_raft_coords_f32(nullptr, coords1, hx.f(), 384, 382, B, h8, w8, st));
      else PP_TRY(pp_k_raft_coords_init(coords1, flow8, hx.h(), 384, 382, B, h8, w8, st));
      e.launches++;

      for (int it = 0; it < iters; ++it) {
        {
          // algorithmic bytes per query pixel: coords 8 B + 4 levels x 10x10 taps + 324 outputs (fp32: hi and lo)
          PPProfScope ps(e, "corr_lookup", (double)M, 0.0, (double)M * (8 + 4 * 100 * cb + 324 * (fp32 ? 8 : 2)), st);
          if (fp32)
            PP_TRY(pp_k_corr_lookup_f32(static_cast<float*>(corr[0]), static_cast<float*>(corr[1]),
                                        static_cast<float*>(corr[2]), static_cast<float*>(corr[3]), coords1,
                                        lk.f(), lk_C, M, h8, w8, st));
          else
            PP_TRY(pp_k_corr_lookup(static_cast<__half*>(corr[0]), static_cast<__half*>(corr[1]),
                                    static_cast<__half*>(corr[2]), static_cast<__half*>(corr[3]), coords1, lk.h(),
                                    lk_C, M, P, h8, w8, st));
        }
        e.launches++;
        // BasicMotionEncoder (update.py:94-112)
        PP_TRY(RConv(e, fp32, "raft.update.convc1", B, h8, w8).in(lk, 0, lk_C).geom(1, 1, 0, 0).out(c1, 0)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(RConv(e, fp32, "raft.update.convc2", B, h8, w8).in(c1, 0, 256).out(corflo, 0).act(PP_ACT_RELU).run(st));
        // convf1 (7x7 over the 2-channel flow): explicit 98-wide patches + a K = 128 linear layer
        if (fp32) PP_TRY(pp_k_flow_patch7x7_f32(coords1, fpatch.f(), B, h8, w8, st));
        else PP_TRY(pp_k_flow_patch7x7(flow8, fpatch.h(), B, h8, w8, st));
        e.launches++;
        PP_TRY(RConv(e, fp32, "raft.update.convf1", 1, 1, (int)M).in(fpatch, 0, 128).geom(1, 1, 0, 0).out(f1b, 0)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(RConv(e, fp32, "raft.update.convf2", B, h8, w8).in(f1b, 0, 128).out(corflo, 192).act(PP_ACT_RELU).run(st));
        PP_TRY(RConv(e, fp32, "raft.update.conv", B, h8, w8).in(corflo, 0, 256).out(hx, 256).act(PP_ACT_RELU).run(st));
        // SepConvGRU (update.py:35-73): horizontal (1x5) then vertical (5x1)
        for (int half = 1; half <= 2; ++half) {
          const std::string s = std::to_string(half);
          PP_TRY(RConv(e, fp32, "raft.update.gru.zr" + s, B, h8, w8).in(hx, 0, 384).out(z, 0).gru_zr(hx, 0, rh, 0).run(st));
          PP_TRY(RConv(e, fp32, "raft.update.gru.q" + s, B, h8, w8).in(rh, 0, 128).in(hx, 128, 256).out(hx, 0)
                     .gru_h(hx, 0, z, 0).run(st));
        }
        // FlowHead (update.py:6-14)
        PP_TRY(RConv(e, fp32, "raft.update.fh1", B, h8, w8).in(hx, 0, 128).out(fh, 0).act(PP_ACT_RELU).run(st));
        PP_TRY(RConv(e, fp32, "raft.update.fh2", B, h8, w8).in(fh, 0, 256).out_plain_f32(delta, 2).run(st));   // 256 -> 2
        if (fp32) PP_TRY(pp_k_raft_coords_f32(delta, coords1, hx.f(), 384, 382, B, h8, w8, st));
        else PP_TRY(pp_k_raft_coords_update(delta, coords1, flow8, hx.h(), 384, 382, B, h8, w8, st));
        e.launches++;
      }
      // mask head (x0.25) + convex upsampling, last iteration only
      {
        Act mk;
        PP_TRY(alloc_act(e, fp32, mk, M, 576, "upsample mask"));
        PP_TRY(RConv(e, fp32, "raft.update.mask0", B, h8, w8).in(hx, 0, 128).out(fh, 0).act(PP_ACT_RELU).run(st));
        PP_TRY(RConv(e, fp32, "raft.update.mask2", B, h8, w8).in(fh, 0, 256).geom(1, 1, 0, 0).out(mk, 0)
                   .act(PP_ACT_NONE, 0.f, 0.25f).run(st));
        for (int si = 0; si < nsub; ++si) {
          const Sub& sb = subs[si];
          float* dst = (sb.dir == 0 ? flows_f : flows_b) + (size_t)sb.b0 * 2 * H * W;
          const float* c1p = coords1 + (size_t)sb.off * P * 2;
          if (fp32) PP_TRY(pp_k_convex_upsample_f32(c1p, mk.f() + (size_t)sb.off * P * 1152, dst, sb.cnt, h8, w8, st));
          else PP_TRY(pp_k_convex_upsample(c1p, mk.h() + (size_t)sb.off * P * 576, dst, sb.cnt, h8, w8, st));
          e.launches++;
        }
      }
      e.arena.release(m2);
    }
  }
  e.arena.release(mark0);
  return PP_OK;
}

// Stage 1: bidirectional RAFT optical flow (reference: model/modules/flow_comp_raft.py:39-58,
// model/modules/RAFT/raft.py:94-152).  Result-identical restructuring vs the reference:
//   * fnet / cnet run once per frame (InstanceNorm is per-sample, BatchNorm is in eval mode), not once per
//     pair and direction;
//   * all pairs of both directions are batched (pairs are independent), bounded only by workspace;
//   * the mask head and convex upsampling run only after the last GRU iteration (raft.py:141-150 keeps
//     only the last flow_up).
// Two precisions share this code, chosen by the element type E the stage is instantiated with.  __half: fp16 activations
// and correlation pyramid, fp32 accumulation.  float (the node's fp16="disable"): every activation is an fp32 split-tf32
// pair tensor [pix][hi C | lo C] and every convolution and the correlation GEMM run as 3xTF32 (conv_igemm.cuh), the
// pyramid is fp32; only the accumulation order differs from fp32.
#include <string.h>

#include "engine.cuh"

namespace {

// What differs between the two precisions, apart from the element type itself
template <class E>
struct Prec {
  static constexpr bool f32 = sizeof(E) == 4;
  static constexpr int act_el = f32 ? 2 : 1;          // elements of E per activation channel (fp32: hi and lo)
  static constexpr int in_C = f32 ? 4 : 8;            // input frames: 3 channels + zeros up to a 16-byte vector
  // lookup output: 324 channels padded to 328 (fp16) / 352 (fp32: 32-channel K chunks of the split segments)
  static constexpr int lk_C = f32 ? 352 : 328;
  static constexpr int corr_K = f32 ? 3 * 256 : 256;  // K of the correlation GEMM (fp32: the segments (hi, lo, hi))
  // launches of one instance norm: memset + statistics + apply (fp32: the statistics take two passes)
  static constexpr int norm_launches = f32 ? 5 : 3;
  static constexpr const char* weights = f32 ? ".tf32" : "";   // suffix of a layer's weight image (engine.py)
};

// An activation tensor of the stage's precision: fp16 [pix][C], or (fp32) a split pair tensor float [pix][hi C | lo C].
template <class E>
struct Act {
  E* p;
  int C;
  Act at(long long pixel) const { return Act{p + pixel * C * Prec<E>::act_el, C}; }
};

template <class E>
int alloc_act(PPEngine& e, Act<E>& a, long long pixels, int C, const char* what) {
  a.C = C;
  return pp_alloc(e, &a.p, (size_t)pixels * C * Prec<E>::act_el, what);
}

// One convolution in the stage's precision.  The builder's channel offsets and counts are real channels in both.
template <class E>
PPConvCall conv(PPEngine& e, const std::string& name, int N, int H, int W) {
  return PPConvCall(e, name + Prec<E>::weights, N, H, W);
}

struct Enc {
  PPEngine& e;
  cudaStream_t st;
  std::string pre;  // "raft.fnet." / "raft.cnet."
  bool inst;
  float* sums;      // [n][2][C] scratch for instance norm
};

// conv (+ instance norm or folded batch norm) (+ relu) (+ residual, relu)
template <class E>
int enc_conv(Enc& c, const std::string& name, const Act<E>& x, int n, int H, int W, int stride, const Act<E>& out,
             bool relu, const Act<E>* residual) {
  PPConvCall call = conv<E>(c.e, c.pre + name, n, H, W);
  call.in(x.p, x.C, 0, x.C);
  const int kh = call.p.kh, kw = call.p.kw;
  call.geom(stride, stride, (kh - 1) / 2, (kw - 1) / 2);
  const int OH = (H + 2 * ((kh - 1) / 2) - (kh - 1) - 1) / stride + 1;
  const int OW = (W + 2 * ((kw - 1) / 2) - (kw - 1) - 1) / stride + 1;
  call.out(out.p, out.C, 0);
  if (c.inst) {
    // raw conv output -> statistics -> normalise in place (+relu, +residual)
    PP_TRY(call.run(c.st));
    PP_TRY(pp_k_instnorm_stats(out.p, n, OH * OW, out.C, c.sums, c.st));
    PP_TRY(pp_k_instnorm_apply(out.p, c.sums, residual ? residual->p : nullptr, out.p, n, OH * OW, out.C, relu ? 1 : 0,
                               c.st));
    c.e.launches += Prec<E>::norm_launches;
  } else {
    if (residual != nullptr)
      call.act(relu ? PP_ACT_RELU : PP_ACT_NONE, 0.f, 1.f, PP_ACT_RELU).residual(residual->p, residual->C, 0);
    else call.act(relu ? PP_ACT_RELU : PP_ACT_NONE);
    PP_TRY(call.run(c.st));
  }
  return PP_OK;
}

// BasicEncoder on n frames: x [n][H][W][x.C] -> out [n][H/8][W/8][256]
template <class E>
int encoder(Enc& c, const Act<E>& x, int n, int H, int W, const Act<E>& out) {
  PPEngine& e = c.e;
  const size_t mark = e.arena.mark();
  const int h2 = (H + 2 * 3 - 7) / 2 + 1, w2 = (W + 2 * 3 - 7) / 2 + 1;
  const long long px = (long long)n * h2 * w2;
  Act<E> a, b, y;
  PP_TRY(alloc_act(e, a, px, 64, "raft enc a"));
  PP_TRY(alloc_act(e, b, px, 64, "raft enc b"));
  PP_TRY(alloc_act(e, y, px, 64, "raft enc y"));
  PP_TRY(enc_conv<E>(c, "conv1", x, n, H, W, 2, a, true, nullptr));
  Act<E> cur = a, nxt = b;
  int hh = h2, ww = w2;
  const int dims[3] = {64, 96, 128};
  for (int li = 0; li < 3; ++li) {
    for (int bi = 0; bi < 2; ++bi) {
      const int s = (li > 0 && bi == 0) ? 2 : 1;
      const int co = dims[li];
      const std::string q = "layer" + std::to_string(li + 1) + "." + std::to_string(bi) + ".";
      const int oh = (hh + 2 - 3) / s + 1, ow = (ww + 2 - 3) / s + 1;
      // the buffers hold 64 channels at h2 x w2: every later layer has at most as many values per image
      Act<E> y1{y.p, co}, nx{nxt.p, co}, cu{cur.p, co};
      // y1 = relu(norm1(conv1(x)))
      PP_TRY(enc_conv<E>(c, q + "conv1", cur, n, hh, ww, s, y1, true, nullptr));
      if (s != 1) {
        // x = norm3(downsample(x)) -- written into nxt first, then used as the residual of conv2 in place
        PP_TRY(enc_conv<E>(c, q + "downsample", cur, n, hh, ww, s, nx, false, nullptr));
        // out = relu(x + relu(norm2(conv2(y1)))) -> needs a third buffer: reuse `cur` (its content is dead now)
        PP_TRY(enc_conv<E>(c, q + "conv2", y1, n, oh, ow, 1, cu, true, &nx));
        cur = cu;   // result is in cur
      } else {
        PP_TRY(enc_conv<E>(c, q + "conv2", y1, n, oh, ow, 1, nx, true, &cur));
        nxt = cur;
        cur = nx;
      }
      hh = oh; ww = ow;
    }
  }
  PP_TRY(conv<E>(e, c.pre + "conv2", n, hh, ww).in(cur.p, cur.C, 0, cur.C).geom(1, 1, 0, 0).out(out.p, out.C, 0).run(c.st));
  e.arena.release(mark);
  return PP_OK;
}

}  // namespace

int pp_raft_corr_pad(int P) {
  const int ntile = pp_ceil_div(P, 256);
  return ((pp_ceil_div(P, ntile) + 15) / 16) * 16 * ntile;
}

template <class E>
int pp_raft_corr_volume(PPEngine& e, const E* fmap1, const E* fpack2, int pairs, int P, int P_pad, E* corr0,
                        cudaStream_t st) {
  // all-pairs correlation: grouped GEMM, one group per frame pair, scaled by 1/sqrt(256)
  PP_REQUIRE((long long)P * P < (1LL << 31), "raft: frame too large for the correlation volume indexing");
  constexpr size_t cb = sizeof(E);
  constexpr int fk = Prec<E>::corr_K;
  const long long Ms = (long long)pairs * P;
  PPConvParams p;
  memset(&p, 0, sizeof(p));
  if constexpr (Prec<E>::f32) {
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
    p.seg[0].ptr = fmap1; p.seg[0].cstride = 256; p.seg[0].coff = 0;
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
  p.out = corr0; p.out_cstride = P; p.out_coff = 0; p.out_fp32 = Prec<E>::f32 ? 1 : 0;
  p.out_gstep = P * P;
  {
    PPProfScope ps(e, "conv:igemm:raft.corr", (double)Ms, 2.0 * Ms * P * fk, (double)Ms * P * cb + 2.0 * Ms * fk * cb, st);
    PP_TRY(pp_launch_conv(p, st));
  }
  e.launches++;
  return PP_OK;
}
template int pp_raft_corr_volume(PPEngine&, const __half*, const __half*, int, int, int, __half*, cudaStream_t);
template int pp_raft_corr_volume(PPEngine&, const float*, const float*, int, int, int, float*, cudaStream_t);

template <class E>
int pp_raft_corr_pool(PPEngine& e, E* const corr[4], long long M, int h8, int w8, cudaStream_t st) {
  for (int l = 0; l < 3; ++l) {
    PP_TRY(pp_k_corr_pool(corr[l], corr[l + 1], M, h8 >> l, w8 >> l, st));
    e.launches++;
  }
  return PP_OK;
}
template int pp_raft_corr_pool(PPEngine&, __half* const*, long long, int, int, cudaStream_t);
template int pp_raft_corr_pool(PPEngine&, float* const*, long long, int, int, cudaStream_t);

template <class E>
int pp_stage_raft(PPEngine& e, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                  cudaStream_t st) {
  PP_REQUIRE(T >= 2, "raft: need at least 2 frames, got %d", T);
  PP_REQUIRE(H % 8 == 0 && W % 8 == 0, "raft: size %dx%d must be a multiple of 8", W, H);
  PP_REQUIRE((H / 8) >= 16 && (W / 8) >= 16, "raft: H/8 and W/8 must be >= 16 (4-level correlation pyramid)");
  using Pr = Prec<E>;
  constexpr bool F32 = Pr::f32;
  constexpr size_t cb = sizeof(E);                   // bytes per correlation value / per packed fmap value
  constexpr size_t ab = Pr::act_el * sizeof(E);      // bytes per activation channel
  constexpr int fk = Pr::corr_K, lk_C = Pr::lk_C;
  const int h8 = H / 8, w8 = W / 8, P = h8 * w8;
  const size_t mark0 = e.arena.mark();

  // ---- per-frame encoders ------------------------------------------------------------------------
  Act<E> fmap, cmap;
  E* fpack;
  const int P_pad = pp_raft_corr_pad(P);
  PP_TRY(alloc_act(e, fmap, (long long)T * P, 256, "fmap"));
  PP_TRY(alloc_act(e, cmap, (long long)T * P, 256, "cmap"));
  PP_TRY(pp_alloc(e, &fpack, (size_t)T * P_pad * fk, "fmap packed"));
  {
    const size_t m1 = e.arena.mark();
    const long long half_px = (long long)(H / 2) * (W / 2);
    int chunk = (int)((8LL << 20) / half_px);
    if (chunk < 1) chunk = 1;
    if (chunk > T) chunk = T;
    Act<E> x;
    float* sums;
    PP_TRY(alloc_act(e, x, (long long)chunk * H * W, Pr::in_C, "raft input"));
    PP_TRY(pp_alloc(e, &sums, pp_k_instnorm_scratch_floats(chunk, (H / 2) * (W / 2), 256), "instnorm sums"));
    for (int f0 = 0; f0 < T; f0 += chunk) {
      const int n = (f0 + chunk <= T) ? chunk : T - f0;
      PP_TRY(pp_k_nchw_to_act(frames + (size_t)f0 * 3 * H * W, x.p, n, 3, H, W, x.C, st));
      e.launches++;
      Enc fe{e, st, "raft.fnet.", true, sums};
      PP_TRY(encoder(fe, x, n, H, W, fmap.at((long long)f0 * P)));
      Enc ce{e, st, "raft.cnet.", false, sums};
      PP_TRY(encoder(ce, x, n, H, W, cmap.at((long long)f0 * P)));
    }
    e.arena.release(m1);
  }
  PP_TRY(pp_k_pack_b_operand(fmap.p, fpack, T, P, P_pad, 256, st));
  e.launches++;

  // ---- pair batches -----------------------------------------------------------------------------
  const int lvl_h[4] = {h8, h8 >> 1, h8 >> 2, h8 >> 3}, lvl_w[4] = {w8, w8 >> 1, w8 >> 2, w8 >> 3};
  size_t corr_elems = 0;
  for (int l = 0; l < 4; ++l) corr_elems += (size_t)P * lvl_h[l] * lvl_w[l];
  // per pair: pyramid, activations (hx rh z lk c1 corflo f1 patches fh), fp16: flow8, coords + delta, slack, mask
  const size_t per_pair = corr_elems * cb + (size_t)P * (384 + 128 + 128 + lk_C + 256 + 256 + 128 + 128 + 256) * ab +
                          (F32 ? 0 : (size_t)P * 8 * 2) + (size_t)P * 4 * 4 + (size_t)P * 32 * 4 + (size_t)P * 576 * ab;
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
      E* corr[4];
      for (int l = 0; l < 4; ++l) PP_TRY(pp_alloc(e, &corr[l], (size_t)M * lvl_h[l] * lvl_w[l], "corr level"));
      for (int si = 0; si < nsub; ++si) {
        const Sub& sb = subs[si];
        const int f1 = sb.dir == 0 ? sb.b0 : sb.b0 + 1;  // first frame playing image1
        const int f2 = sb.dir == 0 ? sb.b0 + 1 : sb.b0;  // first frame playing image2
        PP_TRY(pp_raft_corr_volume<E>(e, fmap.at((long long)f1 * P).p, fpack + (size_t)f2 * P_pad * fk, sb.cnt, P, P_pad,
                                      corr[0] + (size_t)sb.off * P * P, st));
      }
      PP_TRY(pp_raft_corr_pool(e, corr, M, h8, w8, st));
      // GRU state and scratch
      Act<E> hx, rh, z, lk, c1, corflo, f1b, fpatch, fh;
      __half* flow8 = nullptr;                 // fp16 only: the flow for the 7x7 patches (fp32 takes it from coords1)
      float *coords1, *delta;
      PP_TRY(alloc_act(e, hx, M, 384, "hx"));
      PP_TRY(alloc_act(e, rh, M, 128, "rh"));
      PP_TRY(alloc_act(e, z, M, 128, "z"));
      PP_TRY(alloc_act(e, lk, M, lk_C, "corr lookup"));
      PP_TRY(alloc_act(e, c1, M, 256, "c1"));
      PP_TRY(alloc_act(e, corflo, M, 256, "corflo"));
      PP_TRY(alloc_act(e, f1b, M, 128, "f1"));
      PP_TRY(alloc_act(e, fpatch, M, 128, "flow patches"));
      if (!F32) PP_TRY(pp_alloc(e, &flow8, (size_t)M * 8, "flow8"));
      PP_TRY(alloc_act(e, fh, M, 256, "flow head"));
      PP_TRY(pp_alloc(e, &coords1, (size_t)M * 2, "coords1"));
      PP_TRY(pp_alloc(e, &delta, (size_t)M * 2, "delta"));
      // coords1 = coords0 (d == nullptr) or coords1 + d, and the flow into the GRU input
      auto coords = [&](const float* d) {
        if constexpr (F32) return pp_k_raft_coords(d, coords1, hx.p, hx.C, 382, B, h8, w8, st);
        else return pp_k_raft_coords(d, coords1, flow8, hx.p, hx.C, 382, B, h8, w8, st);
      };
      const E* patch_src;                      // what the 7x7 flow patches are cut from
      if constexpr (F32) patch_src = coords1;
      else patch_src = flow8;
      for (int si = 0; si < nsub; ++si) {
        const Sub& sb = subs[si];
        const int f1 = sb.dir == 0 ? sb.b0 : sb.b0 + 1;
        PP_TRY(pp_k_cnet_split(cmap.at((long long)f1 * P).p, hx.at((long long)sb.off * P).p, hx.C,
                               (long long)sb.cnt * P, st));
        e.launches++;
      }
      PP_TRY(coords(nullptr));
      e.launches++;

      for (int it = 0; it < iters; ++it) {
        {
          // algorithmic bytes per query pixel: coords 8 B + 4 levels x 10x10 taps + 324 outputs (fp32: hi and lo)
          PPProfScope ps(e, "corr_lookup", (double)M, 0.0, (double)M * (8 + 4 * 100 * cb + 324 * ab), st);
          PP_TRY(pp_k_corr_lookup(corr[0], corr[1], corr[2], corr[3], coords1, lk.p, lk_C, M, h8, w8, st));
        }
        e.launches++;
        // BasicMotionEncoder (update.py:94-112)
        PP_TRY(conv<E>(e, "raft.update.convc1", B, h8, w8).in(lk.p, lk.C, 0, lk_C).geom(1, 1, 0, 0).out(c1.p, c1.C, 0)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(conv<E>(e, "raft.update.convc2", B, h8, w8).in(c1.p, c1.C, 0, 256).out(corflo.p, corflo.C, 0)
                   .act(PP_ACT_RELU).run(st));
        // convf1 (7x7 over the 2-channel flow): explicit 98-wide patches + a K = 128 linear layer
        PP_TRY(pp_k_flow_patch7x7(patch_src, fpatch.p, B, h8, w8, st));
        e.launches++;
        PP_TRY(conv<E>(e, "raft.update.convf1", 1, 1, (int)M).in(fpatch.p, fpatch.C, 0, 128).geom(1, 1, 0, 0)
                   .out(f1b.p, f1b.C, 0).act(PP_ACT_RELU).run(st));
        PP_TRY(conv<E>(e, "raft.update.convf2", B, h8, w8).in(f1b.p, f1b.C, 0, 128).out(corflo.p, corflo.C, 192)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(conv<E>(e, "raft.update.conv", B, h8, w8).in(corflo.p, corflo.C, 0, 256).out(hx.p, hx.C, 256)
                   .act(PP_ACT_RELU).run(st));
        // SepConvGRU (update.py:35-73): horizontal (1x5) then vertical (5x1)
        for (int half = 1; half <= 2; ++half) {
          const std::string s = std::to_string(half);
          PP_TRY(conv<E>(e, "raft.update.gru.zr" + s, B, h8, w8).in(hx.p, hx.C, 0, 384).out(z.p, z.C, 0)
                     .gru_zr(hx.p, hx.C, 0, rh.p, rh.C, 0).run(st));
          PP_TRY(conv<E>(e, "raft.update.gru.q" + s, B, h8, w8).in(rh.p, rh.C, 0, 128).in(hx.p, hx.C, 128, 256)
                     .out(hx.p, hx.C, 0).gru_h(hx.p, hx.C, 0, z.p, z.C, 0).run(st));
        }
        // FlowHead (update.py:6-14)
        PP_TRY(conv<E>(e, "raft.update.fh1", B, h8, w8).in(hx.p, hx.C, 0, 128).out(fh.p, fh.C, 0).act(PP_ACT_RELU).run(st));
        PP_TRY(conv<E>(e, "raft.update.fh2", B, h8, w8).in(fh.p, fh.C, 0, 256).out_f32(delta, 2, 0).run(st));   // 256 -> 2
        PP_TRY(coords(delta));
        e.launches++;
      }
      // mask head (x0.25) + convex upsampling, last iteration only
      {
        Act<E> mk;
        PP_TRY(alloc_act(e, mk, M, 576, "upsample mask"));
        PP_TRY(conv<E>(e, "raft.update.mask0", B, h8, w8).in(hx.p, hx.C, 0, 128).out(fh.p, fh.C, 0).act(PP_ACT_RELU).run(st));
        PP_TRY(conv<E>(e, "raft.update.mask2", B, h8, w8).in(fh.p, fh.C, 0, 256).geom(1, 1, 0, 0).out(mk.p, mk.C, 0)
                   .act(PP_ACT_NONE, 0.f, 0.25f).run(st));
        for (int si = 0; si < nsub; ++si) {
          const Sub& sb = subs[si];
          float* dst = (sb.dir == 0 ? flows_f : flows_b) + (size_t)sb.b0 * 2 * H * W;
          const float* c1p = coords1 + (size_t)sb.off * P * 2;
          PP_TRY(pp_k_convex_upsample(c1p, mk.at((long long)sb.off * P).p, dst, sb.cnt, h8, w8, st));
          e.launches++;
        }
      }
      e.arena.release(m2);
    }
  }
  e.arena.release(mark0);
  return PP_OK;
}
template int pp_stage_raft<__half>(PPEngine&, const float*, int, int, int, int, float*, float*, cudaStream_t);
template int pp_stage_raft<float>(PPEngine&, const float*, int, int, int, int, float*, float*, cudaStream_t);

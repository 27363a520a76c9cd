// Stage 1: bidirectional RAFT optical flow (reference: model/modules/flow_comp_raft.py:39-58,
// model/modules/RAFT/raft.py:94-152).  Result-identical restructuring vs the reference:
//   * fnet / cnet run once per frame (InstanceNorm is per-sample, BatchNorm is in eval mode), not once per
//     pair and direction;
//   * all pairs of both directions are batched (pairs are independent), bounded only by workspace;
//   * the mask head and convex upsampling run only after the last GRU iteration (raft.py:141-150 keeps
//     only the last flow_up).
#include <string.h>

#include "engine.cuh"

namespace {

struct Enc {
  PPEngine& e;
  cudaStream_t st;
  std::string pre;  // "raft.fnet." / "raft.cnet."
  bool inst;
  float* sums;      // [n][2][C] scratch for instance norm
};

// conv (+ instance norm or folded batch norm) (+ relu) (+ residual, relu)
int enc_conv(Enc& c, const std::string& name, const __half* x, int n, int H, int W, int Cin, int stride, __half* out,
             int Cout, bool relu, const __half* residual) {
  PPConvCall call(c.e, c.pre + name, n, H, W);
  call.in(x, Cin, 0, Cin);
  const PPPackedConv* w = nullptr;
  PP_TRY(pp_get_conv(c.e, c.pre + name, &w));
  call.geom(stride, stride, (w->kh - 1) / 2, (w->kw - 1) / 2);
  const int OH = (H + 2 * ((w->kh - 1) / 2) - (w->kh - 1) - 1) / stride + 1;
  const int OW = (W + 2 * ((w->kw - 1) / 2) - (w->kw - 1) - 1) / stride + 1;
  if (c.inst) {
    // raw conv output -> statistics -> normalise in place (+relu, +residual)
    call.out(out, Cout, 0);
    PP_TRY(call.run(c.st));
    PP_TRY(pp_k_instnorm_stats(out, n, OH * OW, Cout, c.sums, c.st));
    PP_TRY(pp_k_instnorm_apply(out, c.sums, residual, out, n, OH * OW, Cout, relu ? 1 : 0, c.st));
    c.e.launches += 3;  // memset + 2 kernels
  } else {
    call.out(out, Cout, 0);
    if (residual != nullptr) call.act(relu ? PP_ACT_RELU : PP_ACT_NONE, 0.f, 1.f, PP_ACT_RELU).residual(residual, Cout, 0);
    else call.act(relu ? PP_ACT_RELU : PP_ACT_NONE);
    PP_TRY(call.run(c.st));
  }
  return PP_OK;
}

// BasicEncoder on n frames: x8 [n][H][W][8] -> out [n][H/8][W/8][256]
int encoder(Enc& c, const __half* x8, int n, int H, int W, __half* out) {
  PPEngine& e = c.e;
  const size_t mark = e.arena.mark();
  const int h2 = (H + 2 * 3 - 7) / 2 + 1, w2 = (W + 2 * 3 - 7) / 2 + 1;
  __half *a, *b, *y;
  PP_TRY(pp_alloc(e, &a, (size_t)n * h2 * w2 * 64, "raft enc a"));
  PP_TRY(pp_alloc(e, &b, (size_t)n * h2 * w2 * 64, "raft enc b"));
  PP_TRY(pp_alloc(e, &y, (size_t)n * h2 * w2 * 64, "raft enc y"));
  PP_TRY(enc_conv(c, "conv1", x8, n, H, W, 8, 2, a, 64, true, nullptr));
  __half* cur = a;
  __half* nxt = b;
  int ch = 64, hh = h2, ww = w2;
  const int dims[3] = {64, 96, 128};
  for (int li = 0; li < 3; ++li) {
    for (int bi = 0; bi < 2; ++bi) {
      const int s = (li > 0 && bi == 0) ? 2 : 1;
      const int co = dims[li];
      const std::string q = "layer" + std::to_string(li + 1) + "." + std::to_string(bi) + ".";
      const int oh = (hh + 2 - 3) / s + 1, ow = (ww + 2 - 3) / s + 1;
      // y1 = relu(norm1(conv1(x)))
      PP_TRY(enc_conv(c, q + "conv1", cur, n, hh, ww, ch, s, y, co, true, nullptr));
      const __half* res = cur;
      if (s != 1) {
        // x = norm3(downsample(x)) -- written into nxt first, then used as the residual of conv2 in place
        PP_TRY(enc_conv(c, q + "downsample", cur, n, hh, ww, ch, s, nxt, co, false, nullptr));
        res = nxt;
        // out = relu(x + relu(norm2(conv2(y1)))) -> needs a third buffer: reuse `cur` (its content is dead now)
        PP_TRY(enc_conv(c, q + "conv2", y, n, oh, ow, co, 1, cur, co, true, res));
        // result is in cur
      } else {
        PP_TRY(enc_conv(c, q + "conv2", y, n, oh, ow, co, 1, nxt, co, true, res));
        std::swap(cur, nxt);
      }
      ch = co; hh = oh; ww = ow;
    }
  }
  PPConvCall fin(e, c.pre + "conv2", n, hh, ww);
  fin.in(cur, ch, 0, ch).geom(1, 1, 0, 0).out(out, 256, 0);
  PP_TRY(fin.run(c.st));
  e.arena.release(mark);
  return PP_OK;
}

}  // namespace

int pp_stage_raft(PPEngine& e, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                  cudaStream_t st) {
  PP_REQUIRE(T >= 2, "raft: need at least 2 frames, got %d", T);
  PP_REQUIRE(H % 8 == 0 && W % 8 == 0, "raft: size %dx%d must be a multiple of 8", W, H);
  PP_REQUIRE((H / 8) >= 16 && (W / 8) >= 16, "raft: H/8 and W/8 must be >= 16 (4-level correlation pyramid)");
  const int h8 = H / 8, w8 = W / 8, P = h8 * w8;
  const size_t mark0 = e.arena.mark();

  // ---- per-frame encoders ------------------------------------------------------------------------
  __half *fmap, *cmap, *fpack;
  int P_pad;
  {
    const int ntile = pp_ceil_div(P, 256);
    const int bn = ((pp_ceil_div(P, ntile) + 15) / 16) * 16;
    P_pad = bn * ntile;
  }
  PP_TRY(pp_alloc(e, &fmap, (size_t)T * P * 256, "fmap"));
  PP_TRY(pp_alloc(e, &cmap, (size_t)T * P * 256, "cmap"));
  PP_TRY(pp_alloc(e, &fpack, (size_t)T * P_pad * 256, "fmap packed"));
  {
    const size_t m1 = e.arena.mark();
    const long long half_px = (long long)(H / 2) * (W / 2);
    int chunk = (int)((8LL << 20) / half_px);
    if (chunk < 1) chunk = 1;
    if (chunk > T) chunk = T;
    __half* x8;
    float* sums;
    PP_TRY(pp_alloc(e, &x8, (size_t)chunk * H * W * 8, "raft input"));
    PP_TRY(pp_alloc(e, &sums, pp_k_instnorm_scratch_floats(chunk, (H / 2) * (W / 2), 256), "instnorm sums"));
    for (int f0 = 0; f0 < T; f0 += chunk) {
      const int n = (f0 + chunk <= T) ? chunk : T - f0;
      PP_TRY(pp_k_nchw_f32_to_nhwc_f16(frames + (size_t)f0 * 3 * H * W, x8, n, 3, H, W, 8, 0, 8, st));
      e.launches++;
      Enc fe{e, st, "raft.fnet.", true, sums};
      PP_TRY(encoder(fe, x8, n, H, W, fmap + (size_t)f0 * P * 256));
      Enc ce{e, st, "raft.cnet.", false, sums};
      PP_TRY(encoder(ce, x8, n, H, W, cmap + (size_t)f0 * P * 256));
    }
    e.arena.release(m1);
  }
  PP_TRY(pp_k_pack_b_operand(fmap, fpack, T, P, P_pad, 256, st));
  e.launches++;

  // ---- pair batches -----------------------------------------------------------------------------
  const int lvl_h[4] = {h8, h8 >> 1, h8 >> 2, h8 >> 3}, lvl_w[4] = {w8, w8 >> 1, w8 >> 2, w8 >> 3};
  size_t corr_elems = 0;
  for (int l = 0; l < 4; ++l) corr_elems += (size_t)P * lvl_h[l] * lvl_w[l];
  const size_t per_pair = corr_elems * 2 + (size_t)P * (384 + 128 + 128 + 328 + 256 + 256 + 128 + 128 + 8 + 256) * 2 +
                          (size_t)P * 4 * 4 + (size_t)P * 32 * 4 + (size_t)P * 576 * 2;
  const size_t avail = e.arena.cap - e.arena.off;
  int max_pairs = (int)(avail * 9 / 10 / per_pair);
  PP_REQUIRE(max_pairs >= 1, "raft: workspace too small for one frame pair (%zu bytes needed)", per_pair);
  const int npairs = T - 1;
  const int bn_corr = P_pad / pp_ceil_div(P, 256);

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
      __half* corr[4];
      for (int l = 0; l < 4; ++l) PP_TRY(pp_alloc(e, &corr[l], (size_t)M * lvl_h[l] * lvl_w[l], "corr level"));
      // all-pairs correlation: grouped GEMM, one group per frame pair, scaled by 1/sqrt(256)
      PP_REQUIRE((long long)P * P < (1LL << 31), "raft: frame too large for the correlation volume indexing");
      for (int si = 0; si < nsub; ++si) {
        const Sub& sb = subs[si];
        const int f1 = sb.dir == 0 ? sb.b0 : sb.b0 + 1;  // first frame playing image1
        const int f2 = sb.dir == 0 ? sb.b0 + 1 : sb.b0;  // first frame playing image2
        const long long Ms = (long long)sb.cnt * P;
        PPConvParams p;
        memset(&p, 0, sizeof(p));
        p.nseg = 1;
        p.seg[0].ptr = fmap + (size_t)f1 * P * 256; p.seg[0].cstride = 256; p.seg[0].coff = 0;
        p.seg[0].gstep = P * 256; p.seg[0].cbegin = 0; p.seg[0].cend = 256;
        p.N = 1; p.H = 1; p.W = P; p.OH = 1; p.OW = P; p.Cin = 256;
        p.kh = p.kw = 1; p.sh = p.sw = 1; p.dh = p.dw = 1;
        p.wpacked = fpack + (size_t)f2 * P_pad * 256; p.bias = nullptr;
        p.Cout_g = P; p.Cout_g_pad = P_pad; p.BN = bn_corr; p.groups = sb.cnt;
        p.epi = PP_EPI_STD; p.scale = 1.f / 16.f;
        // group g writes rows [g*P, (g+1)*P) of this sub-range: out index = m*out_cstride + out_coff + g*out_gstep + n
        // (P*P exceeds the int range only beyond 46340 pixels at 1/8 res, i.e. 3.7 MPixel frames)
        p.out = corr[0] + (size_t)sb.off * P * P; p.out_cstride = P; p.out_coff = 0; p.out_fp32 = 0;
        p.out_gstep = P * P;
        {
          PPProfScope ps(e, "conv:igemm:raft.corr", (double)Ms, 2.0 * Ms * P * 256, (double)Ms * P * 2 + 2.0 * Ms * 256 * 2, st);
          PP_TRY(pp_launch_conv(p, st));
        }
        e.launches++;
      }
      for (int l = 0; l < 3; ++l) {
        PP_TRY(pp_k_corr_pool(corr[l], corr[l + 1], M, lvl_h[l], lvl_w[l], st));
        e.launches++;
      }
      // GRU state and scratch
      __half *hx, *rh, *z, *lk, *c1, *corflo, *f1b, *flow8, *fh;
      float *coords1, *delta;
      PP_TRY(pp_alloc(e, &hx, (size_t)M * 384, "hx"));
      PP_TRY(pp_alloc(e, &rh, (size_t)M * 128, "rh"));
      PP_TRY(pp_alloc(e, &z, (size_t)M * 128, "z"));
      PP_TRY(pp_alloc(e, &lk, (size_t)M * 328, "corr lookup"));
      PP_TRY(pp_alloc(e, &c1, (size_t)M * 256, "c1"));
      PP_TRY(pp_alloc(e, &corflo, (size_t)M * 256, "corflo"));
      PP_TRY(pp_alloc(e, &f1b, (size_t)M * 128, "f1"));
      __half* fpatch;
      PP_TRY(pp_alloc(e, &fpatch, (size_t)M * 128, "flow patches"));
      PP_TRY(pp_alloc(e, &flow8, (size_t)M * 8, "flow8"));
      PP_TRY(pp_alloc(e, &fh, (size_t)M * 256, "flow head"));
      PP_TRY(pp_alloc(e, &coords1, (size_t)M * 2, "coords1"));
      PP_TRY(pp_alloc(e, &delta, (size_t)M * 2, "delta"));
      for (int si = 0; si < nsub; ++si) {
        const int f1 = subs[si].dir == 0 ? subs[si].b0 : subs[si].b0 + 1;
        PP_TRY(pp_k_cnet_split(cmap + (size_t)f1 * P * 256, hx + (size_t)subs[si].off * P * 384, 384,
                               (long long)subs[si].cnt * P, st));
        e.launches++;
      }
      PP_TRY(pp_k_raft_coords_init(coords1, flow8, hx, 384, 382, B, h8, w8, st));
      e.launches++;

      for (int it = 0; it < iters; ++it) {
        {
          // algorithmic bytes per query pixel: coords 8 B + 4 levels x 10x10 taps x 2 B + 324 outputs x 2 B
          PPProfScope ps(e, "corr_lookup", (double)M, 0.0, (double)M * (8 + 4 * 100 * 2 + 324 * 2), st);
          PP_TRY(pp_k_corr_lookup(corr[0], corr[1], corr[2], corr[3], coords1, lk, 328, M, P, h8, w8, st));
        }
        e.launches++;
        // BasicMotionEncoder (update.py:94-112)
        PP_TRY(PPConvCall(e, "raft.update.convc1", B, h8, w8).in(lk, 328, 0, 328).geom(1, 1, 0, 0)
                   .out(c1, 256, 0).act(PP_ACT_RELU).run(st));
        PP_TRY(PPConvCall(e, "raft.update.convc2", B, h8, w8).in(c1, 256, 0, 256).out(corflo, 256, 0)
                   .act(PP_ACT_RELU).run(st));
        // convf1 (7x7 over the 2-channel flow): explicit 98-wide patches + a K = 128 linear layer
        PP_TRY(pp_k_flow_patch7x7(flow8, fpatch, B, h8, w8, st));
        e.launches++;
        PP_TRY(PPConvCall(e, "raft.update.convf1", 1, 1, (int)M).in(fpatch, 128, 0, 128).geom(1, 1, 0, 0).out(f1b, 128, 0)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(PPConvCall(e, "raft.update.convf2", B, h8, w8).in(f1b, 128, 0, 128).out(corflo, 256, 192)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(PPConvCall(e, "raft.update.conv", B, h8, w8).in(corflo, 256, 0, 256).out(hx, 384, 256)
                   .act(PP_ACT_RELU).run(st));
        // SepConvGRU (update.py:35-73): horizontal (1x5) then vertical (5x1)
        for (int half = 1; half <= 2; ++half) {
          const std::string s = std::to_string(half);
          PP_TRY(PPConvCall(e, "raft.update.gru.zr" + s, B, h8, w8).in(hx, 384, 0, 384).out(z, 128, 0)
                     .gru_zr(hx, 384, 0, rh, 128, 0).run(st));
          PP_TRY(PPConvCall(e, "raft.update.gru.q" + s, B, h8, w8).in(rh, 128, 0, 128).in(hx, 384, 128, 256)
                     .out(hx, 384, 0).gru_h(hx, 384, 0, z, 128, 0).run(st));
        }
        // FlowHead (update.py:6-14)
        PP_TRY(PPConvCall(e, "raft.update.fh1", B, h8, w8).in(hx, 384, 0, 128).out(fh, 256, 0)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(PPConvCall(e, "raft.update.fh2", B, h8, w8).in(fh, 256, 0, 256).out(delta, 2, 0, 1).run(st));   // 256 -> 2, fp32 out
        PP_TRY(pp_k_raft_coords_update(delta, coords1, flow8, hx, 384, 382, B, h8, w8, st));
        e.launches++;
      }
      // mask head (x0.25) + convex upsampling, last iteration only
      {
        __half* mk;
        PP_TRY(pp_alloc(e, &mk, (size_t)M * 576, "upsample mask"));
        PP_TRY(PPConvCall(e, "raft.update.mask0", B, h8, w8).in(hx, 384, 0, 128).out(fh, 256, 0)
                   .act(PP_ACT_RELU).run(st));
        PP_TRY(PPConvCall(e, "raft.update.mask2", B, h8, w8).in(fh, 256, 0, 256).geom(1, 1, 0, 0)
                   .out(mk, 576, 0).act(PP_ACT_NONE, 0.f, 0.25f).run(st));
        for (int si = 0; si < nsub; ++si) {
          const Sub& sb = subs[si];
          float* dst = (sb.dir == 0 ? flows_f : flows_b) + (size_t)sb.b0 * 2 * H * W;
          PP_TRY(pp_k_convex_upsample(coords1 + (size_t)sb.off * P * 2, mk + (size_t)sb.off * P * 576, dst, sb.cnt, h8, w8, st));
          e.launches++;
        }
      }
      e.arena.release(m2);
    }
  }
  e.arena.release(mark0);
  return PP_OK;
}

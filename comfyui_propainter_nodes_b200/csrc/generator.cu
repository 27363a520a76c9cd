// Stage 3b: InpaintGenerator (reference: model/propainter.py:358-453, model/modules/sparse_transformer.py).
//
// Session API: pp_gen_begin() encodes every frame ONCE (the reference re-encodes a frame in every sliding
// window it appears in; the encoder is per-frame, so caching is result-identical) and down-samples flows and
// masks once; pp_gen_run() then runs feature propagation + transformer + decoder for all sliding windows of the clip
// in one batched pass (pp_gen_window(): for a single window), given frame indices into the session.
#include <string.h>

#include "engine.cuh"

namespace {

constexpr int WIN_H = 5, WIN_W = 9, RING = 193;

// 45 own-window token indices followed by the 148 ring tokens of the four rolled copies, in the order of
// valid_ind_rolled (sparse_transformer.py:182-197, 232-283).  Indices address the padded [nh][nw] grid.
}  // namespace

void pp_build_ring_indices(int nh, int nw, std::vector<int>& out) {
  constexpr int WIN_H = 5, WIN_W = 9, RING = 193;
  const int nwh = nh / WIN_H, nww = nw / WIN_W;
  const int eh = (WIN_H + 1) / 2, ew = (WIN_W + 1) / 2;
  out.assign((size_t)nwh * nww * RING, 0);
  for (int wy = 0; wy < nwh; ++wy)
    for (int wx = 0; wx < nww; ++wx) {
      int* dst = &out[((size_t)wy * nww + wx) * RING];
      int n = 0;
      for (int iy = 0; iy < WIN_H; ++iy)
        for (int ix = 0; ix < WIN_W; ++ix) dst[n++] = (wy * WIN_H + iy) * nw + wx * WIN_W + ix;
      // rolled copies: torch.roll(k, shifts=(sy, sx)) => rolled[y][x] = k[(y - sy) mod nh][(x - sx) mod nw]
      const int sy[4] = {-eh, -eh, eh, eh}, sx[4] = {-ew, ew, -ew, ew};
      for (int r = 0; r < 4; ++r)
        for (int iy = 0; iy < WIN_H; ++iy)
          for (int ix = 0; ix < WIN_W; ++ix) {
            const bool top = r < 2, left = (r % 2) == 0;
            // corner masks: tl zero on [:-eh, :-ew]; tr zero on [:-eh, ew:]; bl zero on [eh:, :-ew]; br zero on [eh:, ew:]
            const bool zy = top ? (iy < WIN_H - eh) : (iy >= eh);
            const bool zx = left ? (ix < WIN_W - ew) : (ix >= ew);
            if (zy && zx) continue;
            const int y = ((wy * WIN_H + iy - sy[r]) % nh + nh) % nh;
            const int x = ((wx * WIN_W + ix - sx[r]) % nw + nw) % nw;
            dst[n++] = y * nw + x;
          }
    }
}

namespace {

int deconv(PPEngine& e, const std::string& name, const __half* x, int n, int h, int w, int cin, __half* up,
           __half* out, int cout, int out_cs, int act, float slope, cudaStream_t st) {
  PP_TRY(pp_k_upsample2x(x, cin, 0, up, cin, 0, n, h, w, cin, st));
  e.launches++;
  return PPConvCall(e, name, n, 2 * h, 2 * w).in(up, cin, 0, cin).out(out, out_cs, 0).act(act, slope).run(st);
}

}  // namespace

int pp_stage_gen_end(PPEngine& e) {
  if (e.gen.active) {
    e.arena.release(e.gen.arena_mark);
    e.gen = PPEngine::GenSession();
  }
  return PP_OK;
}

int pp_stage_gen_begin(PPEngine& e, const float* frames, const float* masks_in, const float* masks_upd,
                 const float* flows_f, const float* flows_b, int T, int H, int W, const unsigned char* need,
                 cudaStream_t st) {
  PP_REQUIRE(H % 8 == 0 && W % 8 == 0, "generator: size %dx%d must be a multiple of 8", W, H);
  pp_stage_gen_end(e);
  PPEngine::GenSession& g = e.gen;
  g.arena_mark = e.arena.mark();
  g.active = true;
  g.T = T; g.H = H; g.W = W;
  const int h4 = H / 4, w4 = W / 4, h2 = H / 2, w2 = W / 2;
  const long long P4 = (long long)h4 * w4;
  g.gh = (h4 + 2 * 3 - 7) / 3 + 1;
  g.gw = (w4 + 2 * 3 - 7) / 3 + 1;
  g.nh = pp_ceil_div(g.gh, WIN_H) * WIN_H;
  g.nw = pp_ceil_div(g.gw, WIN_W) * WIN_W;
  g.ph = (g.nh - 4) / 4 + 1;
  g.pw = (g.nw - 4) / 4 + 1;
  PP_TRY(pp_alloc(e, &g.enc, (size_t)T * P4 * 128, "encoder cache"));
  PP_TRY(pp_alloc(e, &g.flows_f4, (size_t)(T - 1) * P4 * 2, "flows_f/4"));
  PP_TRY(pp_alloc(e, &g.flows_b4, (size_t)(T - 1) * P4 * 2, "flows_b/4"));
  PP_TRY(pp_alloc(e, &g.mask_in4, (size_t)T * P4 * 8, "mask2/4"));
  const int n_win = (g.nh / WIN_H) * (g.nw / WIN_W);
  PP_TRY(pp_alloc(e, &g.ring_idx, (size_t)n_win * RING, "ring indices"));
  pp_build_ring_indices(g.nh, g.nw, g.ring_idx_host);
  PP_CUDA_CHECK(cudaMemcpyAsync(g.ring_idx, g.ring_idx_host.data(), g.ring_idx_host.size() * sizeof(int),
                                cudaMemcpyHostToDevice, st));
  // 1/4-res flows (bilinear, /4) and masks (nearest); mask2 = (mask_in, mask_updated, 0 x6) per pixel
  PP_TRY(pp_k_downsample_flow4(flows_f, g.flows_f4, T - 1, H, W, st));
  PP_TRY(pp_k_downsample_flow4(flows_b, g.flows_b4, T - 1, H, W, st));
  PP_CUDA_CHECK(cudaMemsetAsync(g.mask_in4, 0, (size_t)T * P4 * 8 * sizeof(__half), st));
  PP_TRY(pp_k_downsample_mask4(masks_in, g.mask_in4, 8, 0, T, H, W, st));
  PP_TRY(pp_k_downsample_mask4(masks_upd, g.mask_in4, 8, 1, T, H, W, st));
  e.launches += 5;

  // ---- Encoder (propainter.py:234-275) on all frames, in chunks bounded by workspace
  const size_t m1 = e.arena.mark();
  long long per_frame = (long long)H * W * 8 + (long long)h2 * w2 * 64 * 2 + P4 * (128 + 256 + 384 + 512 + 384 + 256);
  long long avail = (long long)(e.arena.cap - e.arena.off) / 2 * 9 / 10;  // elements of fp16
  int chunk = (int)(avail / per_frame);
  if (chunk > T) chunk = T;
  if (chunk > 32) chunk = 32;
  PP_REQUIRE(chunk >= 1, "generator: workspace too small for the encoder");
  __half *x8, *a0, *a1, *a2, *x0, *b8, *b10, *b12, *b14;
  PP_TRY(pp_alloc(e, &x8, (size_t)chunk * H * W * 8, "enc input"));
  PP_TRY(pp_alloc(e, &a0, (size_t)chunk * h2 * w2 * 64, "enc a0"));
  PP_TRY(pp_alloc(e, &a1, (size_t)chunk * h2 * w2 * 64, "enc a1"));
  PP_TRY(pp_alloc(e, &a2, (size_t)chunk * P4 * 128, "enc a2"));
  PP_TRY(pp_alloc(e, &x0, (size_t)chunk * P4 * 256, "enc x0"));
  PP_TRY(pp_alloc(e, &b8, (size_t)chunk * P4 * 384, "enc b8"));
  PP_TRY(pp_alloc(e, &b10, (size_t)chunk * P4 * 512, "enc b10"));
  PP_TRY(pp_alloc(e, &b12, (size_t)chunk * P4 * 384, "enc b12"));
  PP_TRY(pp_alloc(e, &b14, (size_t)chunk * P4 * 256, "enc b14"));
  const long long HW = (long long)H * W;
  // frames to encode: all of them, or (multi-GPU window shards) only the ones this rank's windows touch.  The needed
  // frames are packed into chunks; a chunk is a list of runs of consecutive frames (local frames of a window form one
  // run, the strided reference frames are runs of one).
  std::vector<int> todo;
  for (int f = 0; f < T; ++f)
    if (need == nullptr || need[f]) todo.push_back(f);
  __half* enc_tmp = nullptr;
  if (need != nullptr) PP_TRY(pp_alloc(e, &enc_tmp, (size_t)chunk * P4 * 128, "enc packed output"));
  for (size_t c0 = 0; c0 < todo.size(); c0 += chunk) {
    const int n = (int)((c0 + chunk <= todo.size()) ? chunk : todo.size() - c0);
    struct Run { int frame, slot, len; };
    std::vector<Run> runs;
    for (int i = 0; i < n; ++i) {
      const int f = todo[c0 + i];
      if (!runs.empty() && runs.back().frame + runs.back().len == f) runs.back().len++;
      else runs.push_back(Run{f, i, 1});
    }
    // input = cat(frame[3], mask_in[1], mask_updated[1]) (propainter.py:374-383), padded to 8 channels
    for (const Run& r : runs) {
      __half* dst = x8 + (size_t)r.slot * HW * 8;
      PP_TRY(pp_k_nchw_to_act(frames + (size_t)r.frame * 3 * HW, dst, r.len, 3, H, W, 8, st));
      PP_TRY(pp_k_nchw_to_act(masks_in + (size_t)r.frame * HW, dst, r.len, 1, H, W, 8, st, 3, 1));
      PP_TRY(pp_k_nchw_to_act(masks_upd + (size_t)r.frame * HW, dst, r.len, 1, H, W, 8, st, 4, 1));
      e.launches += 3;
    }
    __half* enc_out = (runs.size() == 1) ? g.enc + (size_t)runs[0].frame * P4 * 128 : enc_tmp;
    const float s = 0.2f;
    PP_TRY(PPConvCall(e, "gen.encoder.0", n, H, W).in(x8, 8, 0, 8).geom(2, 2, 1, 1).out(a0, 64, 0).act(PP_ACT_LRELU, s).run(st));
    PP_TRY(PPConvCall(e, "gen.encoder.2", n, h2, w2).in(a0, 64, 0, 64).out(a1, 64, 0).act(PP_ACT_LRELU, s).run(st));
    PP_TRY(PPConvCall(e, "gen.encoder.4", n, h2, w2).in(a1, 64, 0, 64).geom(2, 2, 1, 1).out(a2, 128, 0).act(PP_ACT_LRELU, s).run(st));
    PP_TRY(PPConvCall(e, "gen.encoder.6", n, h4, w4).in(a2, 128, 0, 128).out(x0, 256, 0).act(PP_ACT_LRELU, s).run(st));
    PP_TRY(PPConvCall(e, "gen.encoder.8", n, h4, w4).in(x0, 256, 0, 256).out(b8, 384, 0).act(PP_ACT_LRELU, s).run(st));
    // grouped layers: group k sees cat(x0[k-th slice], out[k-th slice]) (propainter.py:268-273)
    PP_TRY(PPConvCall(e, "gen.encoder.10", n, h4, w4).in(x0, 256, 0, 128, 128).in(b8, 384, 0, 192, 192)
               .out(b10, 512, 0, 256).act(PP_ACT_LRELU, s).run(st));
    PP_TRY(PPConvCall(e, "gen.encoder.12", n, h4, w4).in(x0, 256, 0, 64, 64).in(b10, 512, 0, 128, 128)
               .out(b12, 384, 0, 96).act(PP_ACT_LRELU, s).run(st));
    // 8 groups of 80 -> 32 channels: dense block-diagonal weights (engine.py), one launch on the halo kernel
    PP_TRY(PPConvCall(e, "gen.encoder.14", n, h4, w4).in(x0, 256, 0, 256).in(b12, 384, 0, 384)
               .out(b14, 256, 0).act(PP_ACT_LRELU, s).run(st));
    PP_TRY(PPConvCall(e, "gen.encoder.16", n, h4, w4).in(x0, 256, 0, 256).in(b14, 256, 0, 256)
               .out(enc_out, 128, 0).act(PP_ACT_LRELU, s).run(st));
    if (runs.size() > 1)
      for (const Run& r : runs)
        PP_CUDA_CHECK(cudaMemcpyAsync(g.enc + (size_t)r.frame * P4 * 128, enc_tmp + (size_t)r.slot * P4 * 128,
                                      (size_t)r.len * P4 * 128 * sizeof(__half), cudaMemcpyDeviceToDevice, st));
  }
  e.arena.release(m1);
  return PP_OK;
}

// All sliding windows of a clip in one pass.  Windows are independent (the reference walks them in a Python
// loop), so every stage is batched across them: feature propagation steps run on all windows of equal local
// length at once, the transformer sees the concatenated token rows of all windows, and the decoder runs on all
// local frames.  frame_ids = concatenation of every window's [local frames..., reference frames...].
int pp_stage_gen_run(PPEngine& e, const int* frame_ids, const int* win_t, const int* win_lt, int n_sw, __half* pred,
                     cudaStream_t st) {
  PPEngine::GenSession& g = e.gen;
  PP_REQUIRE(g.active, "generator: pp_gen_begin was not called");
  PP_REQUIRE(n_sw >= 1, "generator: no windows");
  const int H = g.H, W = g.W, h4 = H / 4, w4 = W / 4, h2 = H / 2, w2 = W / 2;
  const long long P4 = (long long)h4 * w4;
  const int gh = g.gh, gw = g.gw, nh = g.nh, nw = g.nw, ng = gh * gw, np = g.ph * g.pw;
  const int n_win = (nh / WIN_H) * (nw / WIN_W);
  const size_t fsz = (size_t)P4 * 128;

  // ---- schedule bookkeeping (host) ----------------------------------------------------------------
  std::vector<int> foff(n_sw + 1, 0), loff(n_sw + 1, 0), f0(n_sw);
  int t_max = 0;
  for (int w = 0; w < n_sw; ++w) {
    const int t = win_t[w], lt = win_lt[w];
    PP_REQUIRE(lt >= 1 && lt <= t, "generator: window %d has l_t=%d t=%d", w, lt, t);
    // the odd transformer blocks attend to frames 1, 3, ...: a window of one frame leaves its masked 5x9 windows
    // without keys there
    PP_REQUIRE(t >= 2, "generator: window %d has t=%d frames; a window needs at least 2", w, t);
    const int* ids = frame_ids + foff[w];
    for (int i = 0; i < t; ++i) PP_REQUIRE(ids[i] >= 0 && ids[i] < g.T, "generator: frame id out of range");
    for (int i = 1; i < lt; ++i) PP_REQUIRE(ids[i] == ids[0] + i, "generator: local frames must be consecutive");
    f0[w] = ids[0];
    foff[w + 1] = foff[w] + t;
    loff[w + 1] = loff[w] + lt;
    if (t > t_max) t_max = t;
  }
  const int TT = foff[n_sw], LT = loff[n_sw];  // all frames / all local frames of the batch
  // groups of windows with equal local length (uniform step count)
  std::vector<int> lts;
  for (int w = 0; w < n_sw; ++w) {
    bool seen = false;
    for (int v : lts) seen = seen || v == win_lt[w];
    if (!seen) lts.push_back(win_lt[w]);
  }
  // one index table for every gather of this call
  std::vector<int> tab;
  auto push = [&](const std::vector<int>& v) { const int o = (int)tab.size(); tab.insert(tab.end(), v.begin(), v.end()); return o; };
  struct Group { int L, n; std::vector<int> wins; int o_x, o_ff, o_sc_src, o_sc_dst; };
  std::vector<Group> groups;
  for (int L : lts) {
    Group G; G.L = L;
    for (int w = 0; w < n_sw; ++w) if (win_lt[w] == L) G.wins.push_back(w);
    G.n = (int)G.wins.size();
    std::vector<int> ix, ifl;
    for (int k = 0; k < L; ++k) for (int w : G.wins) ix.push_back(f0[w] + k);          // [k][w] <- session frame
    for (int k = 0; k < L - 1; ++k) for (int w : G.wins) ifl.push_back(f0[w] + k);     // [k][w] <- session flow
    G.o_x = push(ix); G.o_ff = push(ifl);
    // scatter of the group's results [k][w] into the window-major slots
    std::vector<int> sc_src, sc_dst;
    for (int k = 0; k < L; ++k)
      for (int j = 0; j < G.n; ++j) { sc_src.push_back(k * G.n + j); sc_dst.push_back(foff[G.wins[j]] + k); }
    G.o_sc_src = push(sc_src); G.o_sc_dst = push(sc_dst);
    groups.push_back(G);
  }
  // refs: window-major slot <- session frame
  std::vector<int> ref_dst, ref_src, loc_rows, sw_f0(f0), sw_lt(win_lt, win_lt + n_sw), sw_t(win_t, win_t + n_sw),
      sw_foff(foff.begin(), foff.end() - 1);
  for (int w = 0; w < n_sw; ++w) {
    for (int i = win_lt[w]; i < win_t[w]; ++i) { ref_dst.push_back(foff[w] + i); ref_src.push_back(frame_ids[foff[w] + i]); }
    for (int k = 0; k < win_lt[w]; ++k) loc_rows.push_back(foff[w] + k);                // local frame -> window-major slot
  }
  const int o_ref_dst = push(ref_dst);
  const int o_ref_src = push(ref_src), o_loc = push(loc_rows), o_f0 = push(sw_f0), o_lt = push(sw_lt), o_t = push(sw_t),
            o_foff = push(sw_foff);

  const size_t mark0 = e.arena.mark();
  int* tab_dev;
  PP_TRY(pp_alloc(e, &tab_dev, tab.size(), "gather table"));
  PP_CUDA_CHECK(cudaMemcpyAsync(tab_dev, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, st));

  __half* encw;  // window-major features [TT][P4][128]
  PP_TRY(pp_alloc(e, &encw, (size_t)TT * fsz, "window features"));

  // ---- learnable bidirectional feature propagation (propainter.py:118-231), per group of equal l_t -------
  for (const Group& G : groups) {
    const size_t mg = e.arena.mark();
    const int L = G.L, n = G.n;
    const size_t slab = (size_t)n * fsz;            // one frame index k over the group's windows
    __half *X, *M2, *FF, *FB, *ob, *of, *cond, *o1, *o2, *offs, *cols, *aligned, *bb;
    PP_TRY(pp_alloc(e, &X, (size_t)L * slab, "featprop x"));
    PP_TRY(pp_alloc(e, &M2, (size_t)L * n * P4 * 8, "featprop masks"));
    PP_TRY(pp_alloc(e, &FF, (size_t)(L > 1 ? L - 1 : 1) * n * P4 * 2, "featprop flows f"));
    PP_TRY(pp_alloc(e, &FB, (size_t)(L > 1 ? L - 1 : 1) * n * P4 * 2, "featprop flows b"));
    PP_TRY(pp_alloc(e, &ob, (size_t)L * slab, "featprop backward"));
    PP_TRY(pp_alloc(e, &of, (size_t)L * slab, "featprop forward"));
    PP_TRY(pp_alloc(e, &cond, (size_t)n * P4 * 264, "featprop cond"));
    PP_TRY(pp_alloc(e, &o1, slab, "featprop o1"));
    PP_TRY(pp_alloc(e, &o2, slab, "featprop o2"));
    PP_TRY(pp_alloc(e, &offs, (size_t)n * P4 * 432, "featprop offsets"));
    PP_TRY(pp_alloc(e, &cols, (size_t)n * P4 * 1152, "featprop dcn columns"));
    PP_TRY(pp_alloc(e, &aligned, slab, "featprop aligned"));
    PP_TRY(pp_alloc(e, &bb, (size_t)L * slab, "featprop tmp"));
    PP_TRY(pp_k_gather_blocks(X, g.enc, tab_dev + G.o_x, (long long)L * n, fsz * 2, st));
    PP_TRY(pp_k_gather_blocks(M2, g.mask_in4, tab_dev + G.o_x, (long long)L * n, P4 * 8 * 2, st));
    PP_TRY(pp_k_gather_blocks(FF, g.flows_f4, tab_dev + G.o_ff, (long long)(L - 1) * n, P4 * 2 * 2, st));
    PP_TRY(pp_k_gather_blocks(FB, g.flows_b4, tab_dev + G.o_ff, (long long)(L - 1) * n, P4 * 2 * 2, st));
    e.launches += 4;
    const size_t mslab = (size_t)n * P4 * 8, wslab = (size_t)n * P4 * 2;
    for (int mod = 0; mod < 2; ++mod) {
      const std::string m = mod == 0 ? "gen.fp.backward_1" : "gen.fp.forward_1";
      const __half* src = mod == 0 ? X : ob;  // the forward pass consumes the backward outputs
      __half* dst = mod == 0 ? ob : of;
      for (int i = 0; i < L; ++i) {
        const int idx = mod == 0 ? L - 1 - i : i;
        const __half* cur = src + (size_t)idx * slab;
        const __half* m2 = M2 + (size_t)idx * mslab;
        const __half* prop = cur;
        if (i > 0) {
          const int prev = mod == 0 ? idx + 1 : idx - 1;
          const int fi = mod == 0 ? idx : idx - 1;  // flow index
          const __half* fprop = (mod == 0 ? FF : FB) + (size_t)fi * wslab;
          const __half* fchk = (mod == 0 ? FB : FF) + (size_t)fi * wslab;
          const __half* pprev = dst + (size_t)prev * slab;
          {
            const double px = (double)n * P4;
            PPProfScope ps(e, "featprop_warp", px, 0.0, px * (128 * 2 * 2 + 264 * 2 + 8 + 16), st);
            PP_TRY(pp_k_featprop_cond(cur, 128, pprev, 128, fprop, fchk, m2, 8, cond, 264, n, h4, w4, 128, st));
          }
          e.launches++;
          PP_TRY(PPConvCall(e, m + ".offset.0", n, h4, w4).in(cond, 264, 0, 264).out(o1, 128, 0).act(PP_ACT_LRELU, 0.1f).run(st));
          PP_TRY(PPConvCall(e, m + ".offset.1", n, h4, w4).in(o1, 128, 0, 128).out(o2, 128, 0).act(PP_ACT_LRELU, 0.1f).run(st));
          PP_TRY(PPConvCall(e, m + ".offset.2", n, h4, w4).in(o2, 128, 0, 128).out(o1, 128, 0).act(PP_ACT_LRELU, 0.1f).run(st));
          PP_TRY(PPConvCall(e, m + ".offset.3", n, h4, w4).in(o1, 128, 0, 128).out(offs, 432, 0).run(st));
          // offsets = 3*tanh(.) + flow (dy,dx) (propainter.py:66-68); flow sits at cond[:, 256:258]
          {
            const double px = (double)n * P4;
            PPProfScope ps(e, "dcn_sample", px, 0.0, px * (128 * 2 + 432 * 2 + 1152 * 2), st);
            PP_TRY(pp_k_dcn_sample(pprev, 128, 0, 128, nullptr, 0, 0, 0, offs, 432, cond, 264, 256, 3.0f, cols, n, h4, w4, st));
          }
          e.launches++;
          PP_TRY(PPConvCall(e, m + ".dcn", n, h4, w4).in(cols, 1152, 0, 1152).geom(1, 1, 0, 0).out(aligned, 128, 0).run(st));
          prop = aligned;
        }
        // feat_prop = feat_prop + backbone(cat(cur, feat_prop, mask_current))
        PP_TRY(PPConvCall(e, m + ".backbone.0", n, h4, w4).in(cur, 128, 0, 128).in(prop, 128, 0, 128).in(m2, 8, 0, 8)
                   .out(bb, 128, 0).act(PP_ACT_LRELU, 0.2f).run(st));
        PP_TRY(PPConvCall(e, m + ".backbone.1", n, h4, w4).in(bb, 128, 0, 128).out(dst + (size_t)idx * slab, 128, 0)
                   .residual(prop, 128, 0).run(st));
      }
    }
    // fuse(cat(out_b, out_f, mask)) + x over every (k, window) frame of the group; result reuses `ob`
    PP_TRY(PPConvCall(e, "gen.fp.fuse.0", L * n, h4, w4).in(ob, 128, 0, 128).in(of, 128, 0, 128).in(M2, 8, 0, 8)
               .out(bb, 128, 0).act(PP_ACT_LRELU, 0.2f).run(st));
    PP_TRY(PPConvCall(e, "gen.fp.fuse.1", L * n, h4, w4).in(bb, 128, 0, 128).out(of, 128, 0).residual(X, 128, 0).run(st));
    // scatter [k][w] -> window-major slots: one launch
    PP_TRY(pp_k_copy_blocks(encw, tab_dev + G.o_sc_dst, of, tab_dev + G.o_sc_src, (long long)L * n, fsz * 2, st));
    e.launches++;
    e.arena.release(mg);
  }
  // reference frames straight from the encoder cache: one launch
  PP_TRY(pp_k_copy_blocks(encw, tab_dev + o_ref_dst, g.enc, tab_dev + o_ref_src, (long long)ref_src.size(), fsz * 2, st));
  e.launches++;

  // ---- SoftSplit: unfold(7,3,3) + Linear == 7x7 stride-3 conv (sparse_transformer.py:8-36) ------------
  const long long rows = (long long)TT * ng, rows_pad = (long long)TT * nh * nw;
  __half *x, *xn, *qkv, *pooled, *pkv, *att, *y, *f1, *img40;
  int* flags;
  PP_TRY(pp_alloc(e, &x, (size_t)rows * 512, "tokens"));
  PP_TRY(pp_alloc(e, &xn, (size_t)rows_pad * 512, "normed tokens"));
  PP_TRY(pp_alloc(e, &qkv, (size_t)rows_pad * 1536, "qkv"));
  PP_TRY(pp_alloc(e, &pooled, (size_t)TT * np * 512, "pooled tokens"));
  PP_TRY(pp_alloc(e, &pkv, (size_t)TT * np * 1024, "pooled kv"));
  PP_TRY(pp_alloc(e, &att, (size_t)rows * 512, "attention out"));
  PP_TRY(pp_alloc(e, &y, (size_t)rows * 512, "normed tokens 2"));
  PP_TRY(pp_alloc(e, &f1, (size_t)rows * 1960, "ffn hidden"));
  PP_TRY(pp_alloc(e, &img40, (size_t)TT * P4 * 40, "ffn folded"));
  PP_TRY(pp_alloc(e, &flags, (size_t)n_sw * n_win, "window flags"));
  PP_TRY(PPConvCall(e, "gen.ss", TT, h4, w4).in(encw, 128, 0, 128).geom(3, 3, 3, 3).out(x, 512, 0).run(st));
  if (nh != gh || nw != gw) PP_CUDA_CHECK(cudaMemsetAsync(xn, 0, (size_t)rows_pad * 512 * sizeof(__half), st));
  // window dispatch flags from the local frames' original masks (propainter.py:417-428)
  PP_TRY(pp_k_window_flags(g.mask_in4, 8, 0, tab_dev + o_f0, tab_dev + o_lt, n_sw, h4, w4, gh, gw, nh / WIN_H, nw / WIN_W,
                           flags, st));
  e.launches++;
  // profiling only: how many 5x9 windows of each sliding window are masked (data dependent) -> real attention flops
  std::vector<int> flags_host;
  if (e.profile) {
    flags_host.resize((size_t)n_sw * n_win);
    PP_CUDA_CHECK(cudaMemcpyAsync(flags_host.data(), flags, flags_host.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    PP_CUDA_CHECK(cudaStreamSynchronize(st));
  }

  // gather table scratch of the wgmma attention kernel: [5x9 windows][keys of a masked window]
  const int key_stride = ((t_max + 1) / 2) * (193 + np);
  int* key_tab;
  PP_TRY(pp_alloc(e, &key_tab, (size_t)(nh / WIN_H) * (nw / WIN_W) * key_stride, "attention key table"));

  for (int blk = 0; blk < 8; ++blk) {
    const std::string b = "gen.tf." + std::to_string(blk) + ".";
    const void *g1, *b1, *g2, *b2, *pwt, *pbs;
    PP_TRY(pp_get_tensor(e, b + "norm1.weight", &g1));
    PP_TRY(pp_get_tensor(e, b + "norm1.bias", &b1));
    PP_TRY(pp_get_tensor(e, b + "norm2.weight", &g2));
    PP_TRY(pp_get_tensor(e, b + "norm2.bias", &b2));
    PP_TRY(pp_get_tensor(e, b + "pool.weight", &pwt));
    PP_TRY(pp_get_tensor(e, b + "pool.bias", &pbs));
    PP_TRY(pp_k_layernorm(x, (const float*)g1, (const float*)b1, xn, rows, gh, gw, nh, nw, st));
    PP_TRY(PPConvCall(e, b + "qkv", 1, 1, (int)rows_pad).in(xn, 512, 0, 512).out(qkv, 1536, 0).run(st));
    PP_TRY(pp_k_pool_tokens(xn, (const float*)pwt, (const float*)pbs, pooled, TT, nh, nw, g.ph, g.pw, 512, st));
    PP_TRY(PPConvCall(e, b + "kv", 1, 1, TT * np).in(pooled, 512, 0, 512).out(pkv, 1024, 0).run(st));
    {
      // 4 q k 128 per head and 5x9 window (4 heads): masked windows attend from all t*45 queries to the keys of every
      // 2nd frame (45 own + 148 ring + pooled tokens each), unmasked windows only to the 45 keys of their own frame
      double fl = 0;
      for (int w = 0; e.profile && w < n_sw; ++w) {
        int masked = 0;
        for (int k = 0; k < n_win; ++k) masked += flags_host[(size_t)w * n_win + k] != 0;
        const double q = 45.0 * win_t[w];
        fl += masked * 4.0 * q * ((win_t[w] - blk % 2 + 1) / 2) * (193 + np) * 512;
        fl += (n_win - masked) * 4.0 * q * 45.0 * 512;
      }
      PPProfScope ps(e, "attention", (double)rows_pad, fl, 0.0, st);
      PP_TRY(pp_k_attention(qkv, qkv + 512, qkv + 1024, 1536, pkv, pkv + 512, 1024, att, 512, flags, g.ring_idx,
                            tab_dev + o_foff, tab_dev + o_t, n_sw, t_max, gh, gw, nh, nw, np, blk % 2, key_tab, key_stride,
                            st));
    }
    PP_TRY(PPConvCall(e, b + "proj", 1, 1, (int)rows).in(att, 512, 0, 512).out(x, 512, 0).residual(x, 512, 0).run(st));
    PP_TRY(pp_k_layernorm(x, (const float*)g2, (const float*)b2, y, rows, gh, gw, gh, gw, st));
    // FusionFeedForward (sparse_transformer.py:67-123): fc1 -> fold/normalise/(unfold) -> GELU -> fc2
    PP_TRY(PPConvCall(e, b + "fc1", 1, 1, (int)rows).in(y, 512, 0, 512).out(f1, 1960, 0).run(st));
    {
      PPProfScope ps(e, "fold_ffn", (double)rows, 0.0, (double)rows * 1960 * 2 + (double)TT * P4 * 40 * 2, st);
      PP_TRY(pp_k_fold(f1, 1960, img40, TT, h4, w4, 40, gh, gw, 1, 1, st));
    }
    PP_TRY(PPConvCall(e, b + "fc2", TT, h4, w4).in(img40, 40, 0, 40).geom(3, 3, 3, 3).out(x, 512, 0)
               .residual(x, 512, 0).run(st));
    e.launches += 5;
  }

  // ---- SoftComp on the local frames only (decoder input), + residual (propainter.py:440-451) -----------
  const size_t m2k = e.arena.mark();
  __half *xl, *encl;
  PP_TRY(pp_alloc(e, &xl, (size_t)LT * ng * 512, "local tokens"));
  PP_TRY(pp_alloc(e, &encl, (size_t)LT * fsz, "local features"));
  PP_TRY(pp_k_gather_blocks(xl, x, tab_dev + o_loc, LT, (long long)ng * 512 * 2, st));
  PP_TRY(pp_k_gather_blocks(encl, encw, tab_dev + o_loc, LT, fsz * 2, st));
  e.launches += 2;
  // frames per chunk bounded by the workspace left (SoftComp Linear output + decoder activations)
  const long long HWl = (long long)H * W;
  const long long per_frame = (long long)ng * 6272 + 2 * (long long)fsz + HWl * 64 * 2 + (long long)h2 * w2 * 192;
  long long avail = (long long)(e.arena.cap - e.arena.off) / 2 * 9 / 10;
  int chunk = (int)(avail / per_frame);
  if (chunk > LT) chunk = LT;
  PP_REQUIRE(chunk >= 1, "generator: workspace too small for the decoder");
  __half *sc1, *img128, *encf, *up, *d0, *d1, *d2;
  PP_TRY(pp_alloc(e, &sc1, (size_t)chunk * ng * 6272, "softcomp linear"));
  PP_TRY(pp_alloc(e, &img128, (size_t)chunk * fsz, "softcomp folded"));
  PP_TRY(pp_alloc(e, &encf, (size_t)chunk * fsz, "decoder input"));
  PP_TRY(pp_alloc(e, &up, (size_t)chunk * HWl * 64, "decoder upsampled"));
  PP_TRY(pp_alloc(e, &d0, (size_t)chunk * h2 * w2 * 128, "decoder d0"));
  PP_TRY(pp_alloc(e, &d1, (size_t)chunk * h2 * w2 * 64, "decoder d1"));
  PP_TRY(pp_alloc(e, &d2, (size_t)chunk * HWl * 64, "decoder d2"));
  for (int c0 = 0; c0 < LT; c0 += chunk) {
    const int n = (c0 + chunk <= LT) ? chunk : LT - c0;
    PP_TRY(PPConvCall(e, "gen.sc.embedding", 1, 1, n * ng).in(xl + (size_t)c0 * ng * 512, 512, 0, 512).out(sc1, 6272, 0).run(st));
    PP_TRY(pp_k_fold(sc1, 6272, img128, n, h4, w4, 128, gh, gw, 0, 0, st));
    e.launches++;
    PP_TRY(PPConvCall(e, "gen.sc.bias_conv", n, h4, w4).in(img128, 128, 0, 128).out(encf, 128, 0)
               .residual(encl + (size_t)c0 * fsz, 128, 0).run(st));
    // decoder (propainter.py:304-312) + tanh
    PP_TRY(deconv(e, "gen.decoder.0", encf, n, h4, w4, 128, up, d0, 128, 128, PP_ACT_LRELU, 0.2f, st));
    PP_TRY(PPConvCall(e, "gen.decoder.2", n, h2, w2).in(d0, 128, 0, 128).out(d1, 64, 0).act(PP_ACT_LRELU, 0.2f).run(st));
    PP_TRY(deconv(e, "gen.decoder.4", d1, n, h2, w2, 64, up, d2, 64, 64, PP_ACT_LRELU, 0.2f, st));
    // 64->3 tail + tanh: halo kernel with a 16-column N tile (the input patch is read once, no im2col amplification)
    PP_TRY(PPConvCall(e, "gen.decoder.6", n, H, W).in(d2, 64, 0, 64).out(pred + (size_t)c0 * HWl * 4, 4, 0)
               .act(PP_ACT_TANH).run(st));
  }
  e.arena.release(m2k);
  e.arena.release(mark0);
  return PP_OK;
}

int pp_stage_gen_window(PPEngine& e, const int* frame_ids, int t, int l_t, __half* pred, cudaStream_t st) {
  return pp_stage_gen_run(e, frame_ids, &t, &l_t, 1, pred, st);
}

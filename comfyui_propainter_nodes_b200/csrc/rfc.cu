// Stage 2: recurrent flow completion (reference: model/recurrent_flow_completion.py:315-400,
// propainter_inference.py:102-156).  forward_bidirect_flow runs the same network on the forward flows and on
// the time-flipped backward flows; the two passes are independent, so they are batched here (D = 2 clips),
// which halves the number of serial propagation steps.
//
// Frame order in every buffer is time-major: image index n = t*D + d.  A time slice is then D contiguous
// images (what the propagation convs need), and the (3,1,1) dilation-2 temporal convs of the P3D blocks
// become 2-D convs with kernel (3,1) over an "image" of height Tn and width D*h*w.
#include <stdlib.h>
#include <string.h>

#include "engine.cuh"

namespace {

// The weights of a layer in the stage's precision: E = float uses the split-tf32 images, registered as "<name>.tf32"
// (engine.py)
template <class E>
std::string wn(const std::string& name) {
  return sizeof(E) == sizeof(float) ? name + ".tf32" : name;
}

// P3DBlock (:162-205) followed by the Sequential's LeakyReLU(0.2): spatial 3x3 (stride s) + LReLU, then
// temporal (3,1,1) dilation 2 + LReLU.  Tn frames of D interleaved clips.
template <class E>
int p3d(PPEngine& e, const std::string& name, const E* x, int Tn, int D, int H, int W, int Cin, int stride, int Cout,
        E* tmp, E* out, cudaStream_t st) {
  const int oh = (H + 2 - 3) / stride + 1, ow = (W + 2 - 3) / stride + 1;
  PP_TRY(PPConvCall(e, wn<E>(name + ".conv1"), Tn * D, H, W).in(x, Cin, 0, Cin).geom(stride, stride, 1, 1)
             .out(tmp, Cout, 0).act(PP_ACT_LRELU, 0.2f).run(st));
  PP_TRY(PPConvCall(e, wn<E>(name + ".conv2"), 1, Tn, D * oh * ow).in(tmp, Cout, 0, Cout).geom(1, 1, 2, 0, 2, 1)
             .out(out, Cout, 0).act(PP_ACT_LRELU, 0.2f).run(st));
  return PP_OK;
}

// bilinear x2 of a C-channel activation tensor (fp16 [pix][C] or split [pix][hi C | lo C])
int upsample2x(const __half* src, __half* dst, int N, int H, int W, int C, cudaStream_t st) {
  return pp_k_upsample2x(src, C, 0, dst, C, 0, N, H, W, C, st);
}
int upsample2x(const float* src, float* dst, int N, int H, int W, int C, cudaStream_t st) {
  return pp_k_upsample2x(src, dst, N, H, W, C, st);
}

// cat of three split [pix][hi 128 | lo 128] tensors into one [pix][hi 384 | lo 384] (PPConvCall takes at most two split
// inputs): a pitched copy of the hi rows and one of the lo rows per source
int cat3_split(const float* const src[3], float* dst, long long npix, cudaStream_t st) {
  for (int j = 0; j < 3; ++j)
    for (int part = 0; part < 2; ++part)
      PP_CUDA_CHECK(cudaMemcpy2DAsync(dst + part * 384 + j * 128, 768 * sizeof(float), src[j] + part * 128,
                                      256 * sizeof(float), 128 * sizeof(float), npix, cudaMemcpyDeviceToDevice, st));
  return PP_OK;
}

inline void shard(int n, int parts, int k, int& lo, int& hi) {   // contiguous near-equal split (parallel.py shard_range)
  const int base = n / parts, rem = n % parts;
  lo = k * base + (k < rem ? k : rem);
  hi = lo + base + (k < rem ? 1 : 0);
}

inline bool rfc_use_programs() {
  const char* s = getenv("PP_PROG");
  return s == nullptr || atoi(s) != 0;
}

// Temporal reach of the encoder: four P3D blocks, each a (3,1,1) dilation-2 conv (t-2, t, t+2) => a frame's
// encoding depends on 8 frames either side (recurrent_flow_completion.py:162-205, 252-264).
constexpr int ENC_HALO = 8;

}  // namespace

// team_size >= 2 (ranks [team_first, team_first + team_size) of the communicator make this call together on the same
// inputs): the two direction passes go to the two halves of the team, the per-frame encoder / decoder of a pass is
// sharded over the ranks of its half (encoder with the +-8-frame halo), the serial recurrence runs on every rank of the
// half, and two all-gathers complete the outputs on every rank of the team:
//   encoder features of the half ([Tn][h/8][w/8][128] activations) before the recurrence, completed flows after it.
// E = __half: fp16 activations; the propagation step runs as one multi-layer program (PP_PROG).  E = float (the node's
// fp16="disable"): split-tf32 activations [pix][hi C | lo C] and 3xTF32 convolutions (conv_igemm.cuh), one launch per
// layer, and the owned frames' fusion / decoder / combine run in frame batches sized to the free arena (every output
// pixel keeps its summation order, so the result does not depend on the batch size).
template <class E>
int pp_stage_flow_complete(PPEngine& e, const float* flows_f, const float* flows_b, const float* flow_masks, int T,
                           int H, int W, float* out_f, float* out_b, int team_first, int team_size, cudaStream_t st) {
  PP_REQUIRE(T >= 2, "flow completion: need at least 2 frames");
  PP_REQUIRE(H % 8 == 0 && W % 8 == 0, "flow completion: size %dx%d must be a multiple of 8", W, H);
  constexpr bool F32 = sizeof(E) == sizeof(float);
  constexpr int EPC = F32 ? 2 : 1;              // stored values per channel: split hi | lo, or one fp16
  const int Tn = T - 1;
  const int h2 = H / 2, w2 = W / 2, h4 = H / 4, w4 = W / 4, h8 = H / 8, w8 = W / 8, P = h8 * w8;
  const long long HW = (long long)H * W;
  const size_t mark0 = e.arena.mark();

  // ---- who computes what -------------------------------------------------------------------------
  const bool multi = team_size > 1 && e.comm != nullptr;
  int D = 2, dirs[2] = {0, 1}, G = 1, member = 0;
  const int trank = e.rank - team_first;        // rank inside the team that shares this call
  if (multi) {
    if (trank < 0 || trank >= team_size) return PP_OK;
    G = team_size / 2;
    if (trank >= 2 * G) D = 0;                  // odd team: the last rank only receives
    else { D = 1; dirs[0] = trank / G; member = trank % G; }
  }
  int a = 0, b = Tn;                            // own frames in network time (dir 1: flipped time)
  if (multi && D == 1) shard(Tn, G, member, a, b);
  const int i0 = (a - ENC_HALO > 0) ? a - ENC_HALO : 0, i1 = (b + ENC_HALO < Tn) ? b + ENC_HALO : Tn;
  const int nl = i1 - i0, cnt = b - a;          // encoded frames (with halo), owned frames
  const float* flows_of[2] = {flows_f, flows_b};
  const float* masks_of[2] = {flow_masks, flow_masks + HW};    // forward flows use masks[:-1], backward masks[1:]
  float* out_of[2] = {out_f, out_b};

  const size_t slice = (size_t)(D > 0 ? D : 1) * P * 128 * EPC;  // elements of one time slice
  if (D > 0 && cnt > 0) {
    const int N = nl * D;
    // ---- input: cat(flow*(1-m), m) of network-time frames [i0, i1); backward flows run with flipped time
    // (fp16: 8 channels, 3 used; split: 4 channels, 3 used -- the weights' cin maps, engine.py)
    const int IC = F32 ? 4 : 8;
    E* x8;
    PP_TRY(pp_alloc(e, &x8, (size_t)N * HW * 8, "rfc input"));
    for (int k = 0; k < D; ++k) {
      const int d = dirs[k];
      const int t0 = d == 0 ? i0 : Tn - i1;    // first original-time frame of the range
      PP_TRY(pp_k_rfc_pack_input(flows_of[d] + (size_t)t0 * 2 * HW, masks_of[d] + (size_t)t0 * HW, x8 + (size_t)k * HW * 8,
                                 D * HW, nl, H, W, d, st));
      e.launches++;
    }

    // ---- encoder (on [i0, i1); only [a, b) is exact, the rest is halo) -------------------------------
    E *x, *t1, *e1a, *e1, *e2a, *e2;
    PP_TRY(pp_alloc(e, &x, (size_t)N * h2 * w2 * 32 * EPC, "rfc x"));
    PP_TRY(pp_alloc(e, &t1, (size_t)N * h2 * w2 * 32 * EPC, "rfc tmp"));
    PP_TRY(pp_alloc(e, &e1a, (size_t)N * h2 * w2 * 32 * EPC, "rfc e1a"));
    PP_TRY(pp_alloc(e, &e1, (size_t)N * h4 * w4 * 64 * EPC, "rfc e1"));
    PP_TRY(pp_alloc(e, &e2a, (size_t)N * h4 * w4 * 64 * EPC, "rfc e2a"));
    PP_TRY(pp_alloc(e, &e2, (size_t)N * P * 128 * EPC, "rfc e2"));
    PP_TRY(PPConvCall(e, wn<E>("rfc.downsample"), N, H, W).in(x8, IC, 0, IC).geom(2, 2, 2, 2, 1, 1, 1)
               .out(x, 32, 0).act(PP_ACT_LRELU, 0.2f).run(st));
    PP_TRY(p3d(e, "rfc.encoder1.0", x, nl, D, h2, w2, 32, 1, 32, t1, e1a, st));
    PP_TRY(p3d(e, "rfc.encoder1.2", e1a, nl, D, h2, w2, 32, 2, 64, t1, e1, st));
    PP_TRY(p3d(e, "rfc.encoder2.0", e1, nl, D, h4, w4, 64, 1, 64, t1, e2a, st));
    PP_TRY(p3d(e, "rfc.encoder2.2", e2a, nl, D, h4, w4, 64, 2, 128, t1, e2, st));
    // mid_dilation: three (1,3,3) convs with dilation 3, 2, 1 (:266-280), on the owned frames only; the last one
    // writes into the full-clip feature buffer the recurrence reads
    E *midA, *midB, *mid;
    PP_TRY(pp_alloc(e, &midA, (size_t)cnt * slice, "rfc mid a"));
    PP_TRY(pp_alloc(e, &midB, (size_t)cnt * slice, "rfc mid b"));
    PP_TRY(pp_alloc(e, &mid, (size_t)Tn * slice, "rfc mid"));
    const E* e2own = e2 + (size_t)(a - i0) * slice;
    PP_TRY(PPConvCall(e, wn<E>("rfc.mid.0"), cnt * D, h8, w8).in(e2own, 128, 0, 128).geom(1, 1, 3, 3, 3, 3)
               .out(midA, 128, 0).act(PP_ACT_LRELU, 0.2f).run(st));
    PP_TRY(PPConvCall(e, wn<E>("rfc.mid.1"), cnt * D, h8, w8).in(midA, 128, 0, 128).geom(1, 1, 2, 2, 2, 2)
               .out(midB, 128, 0).act(PP_ACT_LRELU, 0.2f).run(st));
    PP_TRY(PPConvCall(e, wn<E>("rfc.mid.2"), cnt * D, h8, w8).in(midB, 128, 0, 128).geom(1, 1, 1, 1, 1, 1)
               .out(mid + (size_t)a * slice, 128, 0).act(PP_ACT_LRELU, 0.2f).run(st));
    if (multi && G > 1) {
      std::vector<long long> offs(G), rows(G);
      for (int m = 0; m < G; ++m) {
        int lo, hi;
        shard(Tn, G, m, lo, hi);
        offs[m] = lo; rows[m] = hi - lo;
      }
      PP_TRY(pp_comm_all_gather_blocks_impl(e, mid, offs.data(), rows.data(), slice * sizeof(E),
                                            team_first + dirs[0] * G, G, st));
    }

    // ---- bidirectional second-order deformable propagation (:77-143), serial over the whole clip -----------
    // offs and (E = float) pred are plain [pix][C] tensors of E: the sampler / combine read them, no conv does
    E *fb, *ff, *zero, *o1, *o2, *offs, *cols, *aligned, *bb;
    PP_TRY(pp_alloc(e, &fb, (size_t)Tn * slice, "rfc feats backward"));
    PP_TRY(pp_alloc(e, &ff, (size_t)Tn * slice, "rfc feats forward"));
    PP_TRY(pp_alloc(e, &zero, slice, "rfc zeros"));
    PP_TRY(pp_alloc(e, &o1, slice, "rfc o1"));
    PP_TRY(pp_alloc(e, &o2, slice, "rfc o2"));
    PP_TRY(pp_alloc(e, &offs, (size_t)D * P * 432, "rfc offsets"));
    PP_TRY(pp_alloc(e, &cols, (size_t)D * P * 2304 * EPC, "rfc dcn columns"));
    PP_TRY(pp_alloc(e, &aligned, slice, "rfc aligned"));
    PP_TRY(pp_alloc(e, &bb, slice, "rfc backbone tmp"));
    E* cat3 = nullptr;                          // E = float: the three-input layers' materialised concatenation
    if (F32) PP_TRY(pp_alloc(e, &cat3, (size_t)3 * slice, "rfc cat3"));
    PP_CUDA_CHECK(cudaMemsetAsync(zero, 0, slice * sizeof(E), st));
    // One propagation step = 8 dependent layers over D*P pixels (3,600-7,200 at 640x360): as separate launches each
    // costs 15-30 us of mostly fixed overhead, so an fp16 step runs as ONE multi-layer program (conv_halo.cu: persistent
    // CTAs, grid-wide barrier between layers).  PP_PROG=0 falls back to one launch per layer; the programs have no
    // split-tf32 layers, so E = float always runs one launch per layer.
    const bool prog = !F32 && rfc_use_programs();
    struct ProgGuard {      // an error path between begin and end must not leave the recorder armed
      bool armed = false;
      ~ProgGuard() { if (armed) pp_prog_abort(); }
    } pg;
    for (int mod = 0; mod < 2; ++mod) {
      const std::string m = mod == 0 ? "rfc.fp.backward_" : "rfc.fp.forward_";
      E* feats = mod == 0 ? fb : ff;
      for (int i = 0; i < Tn; ++i) {
        if (prog) { PP_TRY(pp_prog_begin()); pg.armed = true; e.prog_flops = 0.0; }
        const int idx = mod == 0 ? Tn - 1 - i : i;
        const int prev = mod == 0 ? idx + 1 : idx - 1, prev2 = mod == 0 ? idx + 2 : idx - 2;
        const E* cur = mid + (size_t)idx * slice;
        const E* prop = zero;
        if (i > 0) {
          const E* p1 = feats + (size_t)prev * slice;
          const E* n2 = i > 1 ? feats + (size_t)prev2 * slice : zero;
          // cond = cat(prop, cur, n2) -> 4-conv offset head (:17-26, 32-42)
          PPConvCall c0(e, wn<E>(m + ".offset.0"), D, h8, w8);
          if constexpr (F32) {
            const float* srcs[3] = {p1, cur, n2};
            PP_TRY(cat3_split(srcs, cat3, (long long)D * P, st));
            c0.in(cat3, 384, 0, 384);
          } else {
            c0.in(p1, 128, 0, 128).in(cur, 128, 0, 128).in(n2, 128, 0, 128);
          }
          PP_TRY(c0.out(o1, 128, 0).act(PP_ACT_LRELU, 0.1f).run(st));
          PP_TRY(PPConvCall(e, wn<E>(m + ".offset.1"), D, h8, w8).in(o1, 128, 0, 128).out(o2, 128, 0)
                     .act(PP_ACT_LRELU, 0.1f).run(st));
          PP_TRY(PPConvCall(e, wn<E>(m + ".offset.2"), D, h8, w8).in(o2, 128, 0, 128).out(o1, 128, 0)
                     .act(PP_ACT_LRELU, 0.1f).run(st));
          PPConvCall c3(e, wn<E>(m + ".offset.3"), D, h8, w8);
          c3.in(o1, 128, 0, 128);
          if constexpr (F32) c3.out_f32(offs, 432, 0);
          else c3.out(offs, 432, 0);
          PP_TRY(c3.run(st));
          // modulated deformable conv on cat(prop, n2): sample -> GEMM (K = 9*256)
          if constexpr (F32) {
            const double px = (double)D * P;
            PPProfScope ps(e, "dcn_sample_f32", px, 0.0, px * (256 * 8 + 432 * 4 + 2304 * 8), st);
            PP_TRY(pp_k_dcn_sample(p1, 128, n2, 128, offs, 432, 5.0f, cols, D, h8, w8, st));
            e.launches++;
          } else if (prog) {
            PP_TRY(pp_k_dcn_sample(p1, 128, 0, 128, n2, 128, 0, 128, offs, 432, nullptr, 0, 0, 5.0f, cols, D, h8, w8, st));
          } else {
            const double px = (double)D * P;
            PPProfScope ps(e, "dcn_sample", px, 0.0, px * (256 * 2 + 432 * 2 + 2304 * 2), st);
            PP_TRY(pp_k_dcn_sample(p1, 128, 0, 128, n2, 128, 0, 128, offs, 432, nullptr, 0, 0, 5.0f, cols, D, h8, w8, st));
            e.launches++;
          }
          PP_TRY(PPConvCall(e, wn<E>(m + ".dcn"), D, h8, w8).in(cols, 2304, 0, 2304).geom(1, 1, 0, 0).out(aligned, 128, 0)
                     .run(st));
          prop = aligned;
        }
        // feat_prop = feat_prop + backbone(cat(cur, [backward feature of this frame], feat_prop))
        PPConvCall b0(e, wn<E>(m + ".backbone.0"), D, h8, w8);
        if constexpr (F32) {
          if (mod == 1) {
            const float* srcs[3] = {cur, fb + (size_t)idx * slice, prop};
            PP_TRY(cat3_split(srcs, cat3, (long long)D * P, st));
            b0.in(cat3, 384, 0, 384);
          } else {
            b0.in(cur, 128, 0, 128).in(prop, 128, 0, 128);
          }
        } else {
          b0.in(cur, 128, 0, 128);
          if (mod == 1) b0.in(fb + (size_t)idx * slice, 128, 0, 128);
          b0.in(prop, 128, 0, 128);
        }
        b0.out(bb, 128, 0).act(PP_ACT_LRELU, 0.1f);
        PP_TRY(b0.run(st));
        PP_TRY(PPConvCall(e, wn<E>(m + ".backbone.1"), D, h8, w8).in(bb, 128, 0, 128)
                   .out(feats + (size_t)idx * slice, 128, 0).residual(prop, 128, 0).run(st));
        if (prog) {
          PPProfScope ps(e, "conv:prog:rfc.fp.step", (double)D * P, e.prog_flops, 0.0, st);
          pg.armed = false;
          PP_TRY(pp_prog_end(e.prog_counter, &e.prog_arrivals, st));
          e.launches++;
        }
      }
    }

    // ---- owned frames [a, b): fusion(cat(backward, forward)) + x (:138-143), decoders (:282-300, 333-345) ---
    const int Nd = cnt * D;
    E* fused = e2;  // e2 is dead
    PP_TRY(PPConvCall(e, wn<E>("rfc.fp.fusion"), Nd, h8, w8).in(fb + (size_t)a * slice, 128, 0, 128)
               .in(ff + (size_t)a * slice, 128, 0, 128).geom(1, 1, 0, 0).out(fused, 128, 0)
               .residual(mid + (size_t)a * slice, 128, 0).run(st));
    // frames per decoder batch: all owned frames for fp16; E = float takes as many as the free arena holds
    int nb = cnt;
    if (F32) {
      const size_t per_img = ((size_t)P * 128 + (size_t)HW * 32 + (size_t)h4 * w4 * 64 * 2 + (size_t)h2 * w2 * 32 * 2) * EPC +
                             (size_t)HW * 2;
      const size_t per_frame = per_img * D * sizeof(E), slack = 7 * 256;
      const size_t free_bytes = e.arena.cap > e.arena.off + slack ? e.arena.cap - e.arena.off - slack : 0;
      const size_t fit = free_bytes / per_frame;
      nb = fit < 1 ? 1 : (fit < (size_t)cnt ? (int)fit : cnt);
    }
    const int Nb = nb * D;
    E *d2a, *up, *d2, *d1a, *d1, *u0, *pred;
    PP_TRY(pp_alloc(e, &d2a, (size_t)Nb * P * 128 * EPC, "rfc d2a"));
    PP_TRY(pp_alloc(e, &up, (size_t)Nb * HW * 32 * EPC, "rfc upsampled"));
    PP_TRY(pp_alloc(e, &d2, (size_t)Nb * h4 * w4 * 64 * EPC, "rfc d2"));
    PP_TRY(pp_alloc(e, &d1a, (size_t)Nb * h4 * w4 * 64 * EPC, "rfc d1a"));
    PP_TRY(pp_alloc(e, &d1, (size_t)Nb * h2 * w2 * 32 * EPC, "rfc d1"));
    PP_TRY(pp_alloc(e, &u0, (size_t)Nb * h2 * w2 * 32 * EPC, "rfc u0"));
    PP_TRY(pp_alloc(e, &pred, (size_t)Nb * HW * 2, "rfc pred"));
    for (int f0 = 0; f0 < cnt; f0 += nb) {
      const int nf = cnt - f0 < nb ? cnt - f0 : nb, Nf = nf * D;
      const E* fz = fused + (size_t)f0 * slice;
      const E* e1own = e1 + (size_t)(a - i0 + f0) * D * h4 * w4 * 64 * EPC;   // skip connection of these frames
      PP_TRY(PPConvCall(e, wn<E>("rfc.decoder2.0"), Nf, h8, w8).in(fz, 128, 0, 128).out(d2a, 128, 0)
                 .act(PP_ACT_LRELU, 0.2f).run(st));
      // deconv = bilinear x2 (materialised in `up`) + 3x3 conv
      PP_TRY(upsample2x(d2a, up, Nf, h8, w8, 128, st));
      PP_TRY(PPConvCall(e, wn<E>("rfc.decoder2.deconv"), Nf, h4, w4).in(up, 128, 0, 128).out(d2, 64, 0)
                 .act(PP_ACT_LRELU, 0.2f).residual(e1own, 64, 0).run(st));
      PP_TRY(PPConvCall(e, wn<E>("rfc.decoder1.0"), Nf, h4, w4).in(d2, 64, 0, 64).out(d1a, 64, 0)
                 .act(PP_ACT_LRELU, 0.2f).run(st));
      PP_TRY(upsample2x(d1a, up, Nf, h4, w4, 64, st));
      PP_TRY(PPConvCall(e, wn<E>("rfc.decoder1.deconv"), Nf, h2, w2).in(up, 64, 0, 64).out(d1, 32, 0)
                 .act(PP_ACT_LRELU, 0.2f).run(st));
      PP_TRY(PPConvCall(e, wn<E>("rfc.upsample.0"), Nf, h2, w2).in(d1, 32, 0, 32).out(u0, 32, 0)
                 .act(PP_ACT_LRELU, 0.2f).run(st));
      PP_TRY(upsample2x(u0, up, Nf, h2, w2, 32, st));
      // 32 -> 2 tail (fp16: channels zero-extended to 64 by TMA, 16-column N tile; E = float: plain fp32 output)
      PPConvCall tail(e, wn<E>("rfc.upsample.deconv"), Nf, H, W);
      tail.in(up, 32, 0, 32);
      if constexpr (F32) tail.out_f32(pred, 2, 0);
      else tail.out(pred, 2, 0);
      PP_TRY(tail.run(st));
      e.launches += 3;

      // ---- combine_flow (:389-400) and un-flip, rows of these frames --------------------------------------
      for (int k = 0; k < D; ++k) {
        const int d = dirs[k];
        const int t0 = d == 0 ? a + f0 : Tn - (a + f0 + nf);      // first original-time frame of the batch
        PP_TRY(pp_k_rfc_combine(pred + (size_t)k * HW * 2, 2, D * HW, flows_of[d] + (size_t)t0 * 2 * HW,
                                masks_of[d] + (size_t)t0 * HW, out_of[d] + (size_t)t0 * 2 * HW, nf, H, W, d, st));
        e.launches++;
      }
    }
  }
  // ---- completed flows of both directions to every rank --------------------------------------------------
  if (multi) {
    for (int d = 0; d < 2; ++d) {
      std::vector<long long> offs(team_size, 0), rows(team_size, 0);
      for (int m = 0; m < G; ++m) {
        int lo, hi;
        shard(Tn, G, m, lo, hi);
        offs[d * G + m] = d == 0 ? lo : Tn - hi;
        rows[d * G + m] = hi - lo;
      }
      PP_TRY(pp_comm_all_gather_blocks_impl(e, out_of[d], offs.data(), rows.data(), (size_t)2 * HW * sizeof(float),
                                            team_first, team_size, st));
    }
  }
  e.arena.release(mark0);
  return PP_OK;
}
template int pp_stage_flow_complete<__half>(PPEngine&, const float*, const float*, const float*, int, int, int, float*,
                                            float*, int, int, cudaStream_t);
template int pp_stage_flow_complete<float>(PPEngine&, const float*, const float*, const float*, int, int, int, float*,
                                           float*, int, int, cudaStream_t);

// Stage 3a: non-learnable image propagation (reference: propainter_inference.py:159-225 single-chunk branch,
// model/propainter.py:118-231 with learnable=False).  One persistent kernel for the 2(T-1) serial steps.  E = float keeps
// frames, masks and flows in fp32 (the node's fp16="disable"): the fb test, the 0.1 mask threshold and the nearest-pixel
// pick are discrete, and an fp16-rounded flow or frame moves whole pixels, not a last bit.
template <class E>
int pp_stage_image_propagate(PPEngine& e, const float* frames, const float* masks, const float* flows_f,
                             const float* flows_b, int T, int H, int W, float* upd_frames, float* upd_masks,
                             cudaStream_t st) {
  PP_REQUIRE(T >= 2, "image propagation: need at least 2 frames");
  const long long HW = (long long)H * W;
  const size_t mark0 = e.arena.mark();
  E *in4, *bwd, *fwd, *ff, *fbk;
  PP_TRY(pp_alloc(e, &in4, (size_t)T * HW * 4, "imgprop input"));
  PP_TRY(pp_alloc(e, &bwd, (size_t)T * HW * 4, "imgprop backward"));
  PP_TRY(pp_alloc(e, &fwd, (size_t)T * HW * 4, "imgprop forward"));
  PP_TRY(pp_alloc(e, &ff, (size_t)(T - 1) * HW * 2, "imgprop flows f"));
  PP_TRY(pp_alloc(e, &fbk, (size_t)(T - 1) * HW * 2, "imgprop flows b"));
  PP_TRY(pp_k_imgprop_pack(frames, masks, in4, T, H, W, st));
  PP_TRY(pp_k_flow_to_nhwc2(flows_f, ff, T - 1, H, W, st));
  PP_TRY(pp_k_flow_to_nhwc2(flows_b, fbk, T - 1, H, W, st));
  e.launches += 3;
  // both passes in one persistent kernel (kernels_prop.cu): bwd / fwd start as copies of the packed input, only the
  // pixels inside the hole's bounding box are touched by the 2(T-1) serial steps
  const size_t all = (size_t)T * HW * 4 * sizeof(E);
  PP_CUDA_CHECK(cudaMemcpyAsync(bwd, in4, all, cudaMemcpyDeviceToDevice, st));
  PP_CUDA_CHECK(cudaMemcpyAsync(fwd, in4, all, cudaMemcpyDeviceToDevice, st));
  int* scratch;
  PP_TRY(pp_alloc(e, &scratch, 8, "imgprop scratch"));
  {
    // algorithmic bytes of the reference's 2(T-1) steps (SURVEY.md 8d: 32 B per pixel and step, fp16); the kernel
    // itself moves far less (hole pixels only + the two up-front copies)
    const double step_bytes = 32.0 * sizeof(E) / sizeof(__half);
    PPProfScope ps(e, sizeof(E) == 4 ? "imgprop_f32" : "imgprop", (double)HW * 2 * (T - 1), 0.0,
                   (double)HW * step_bytes * 2 * (T - 1), st);
    PP_TRY(pp_k_imgprop_run(in4, bwd, fwd, ff, fbk, masks, T, H, W, scratch, st));
  }
  e.launches += 4;
  PP_TRY(pp_k_imgprop_finish(fwd, frames, masks, upd_frames, upd_masks, T, H, W, st));
  e.launches++;
  e.arena.release(mark0);
  return PP_OK;
}
template int pp_stage_image_propagate<__half>(PPEngine&, const float*, const float*, const float*, const float*, int, int,
                                              int, float*, float*, cudaStream_t);
template int pp_stage_image_propagate<float>(PPEngine&, const float*, const float*, const float*, const float*, int, int,
                                             int, float*, float*, cudaStream_t);

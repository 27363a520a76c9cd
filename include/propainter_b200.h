/* C ABI of the H100-native ProPainter inference path (libpropainter_b200.so).
 *
 * Every entry point takes raw device pointers, sizes and a CUDA stream (as void*, 0 = legacy default
 * stream) and returns 0 on success; on failure pp_last_error() holds a message.  No torch types cross this
 * boundary.  Tensors are contiguous, float32, in the layouts the reference's own tensors have at the same
 * call sites (paths relative to daniabib/ComfyUI_ProPainter_Nodes):
 *
 *   pp_raft_bidir[_fp32]   replaces  raft_model(frames, iters)                propainter_inference.py:77-93
 *                                    (RAFT_bi.forward, model/modules/flow_comp_raft.py:39-58)
 *   pp_flow_complete[_fp32] replaces forward_bidirect_flow + combine_flow     propainter_inference.py:123-150
 *                                    (model/recurrent_flow_completion.py:356-400)
 *   pp_image_propagate[_fp32] replaces img_propagation + blend               propainter_inference.py:186-219
 *                                    (model/propainter.py:350-356, 118-231)
 *   pp_gen_begin/window    replace   inpaint_model(selected_imgs, ...)        propainter_inference.py:272-281
 *                                    (InpaintGenerator.forward, model/propainter.py:358-453)
 *   pp_composite           replaces  the numpy composite                      propainter_inference.py:283-307
 *   pp_register_*          replace   load_state_dict of the three checkpoints utils/model_utils.py:49-59
 */
#ifndef PROPAINTER_B200_H
#define PROPAINTER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PP_API __attribute__((visibility("default")))
#else
#define PP_API
#endif

typedef struct PPEngine* pp_handle;

/* Message of the last failing call on this thread. */
PP_API const char* pp_last_error(void);
/* Library build id ("propainter_b200 <n> sm_90a"). */
PP_API const char* pp_version(void);

/* Create an engine on `device` whose scratch arena is the caller-allocated device buffer
 * [workspace, workspace + workspace_bytes) (256-byte aligned). */
PP_API int pp_create(int device, void* workspace, size_t workspace_bytes, pp_handle* out);
PP_API int pp_destroy(pp_handle h);
/* Replace the scratch arena (grow it for a larger clip, or shrink it after one); the previous buffer may be freed by
 * the caller once this returns.  Fails while a generator session is open. */
PP_API int pp_set_workspace(pp_handle h, void* workspace, size_t workspace_bytes);

/* Register packed weights (device memory owned by the caller, must outlive the handle).
 * `w` is the 128B-swizzled tile image produced by comfyui_propainter_nodes_b200.weights_pack,
 * [groups][ceil(kh*kw*cin_g/64)][cout_g_pad] rows of 64 fp16; `bias` is float32 [groups*cout_g] or NULL. */
PP_API int pp_register_conv(pp_handle h, const char* name, const void* w, const float* bias, int cout_g, int cout_g_pad,
                     int bn, int cin_g, int kh, int kw, int groups);
PP_API int pp_register_tensor(pp_handle h, const char* name, const void* ptr, size_t bytes);
/* Multiply-adds per output pixel of the reference layer behind a registered conv (unpadded channels, real groups);
 * only feeds the algorithmic flop count of pp_profile_dump. */
PP_API int pp_set_conv_macs(pp_handle h, const char* name, double macs_per_pixel);

/* ---- multi-GPU: one process per GPU, an NCCL communicator per engine (SURVEY.md 8b/8e) ------------------------
 * Rank 0 calls pp_comm_unique_id and ships the 128 bytes to the other ranks (any host transport); every rank then
 * calls pp_comm_init(h, id, rank, world).  NCCL is resolved with dlopen at run time (the process' own copy first). */
PP_API int pp_comm_unique_id(void* out128);
PP_API int pp_comm_init(pp_handle h, const void* unique_id128, int rank, int world);
PP_API int pp_comm_destroy(pp_handle h);
/* In-place all-gather of uneven row blocks among ranks [first_rank, first_rank + n_members): `buf` holds
 * sum(rows_per_member) rows of row_bytes, member m has written its own block; on return (stream order) every member
 * holds all blocks.  One NCCL send/recv group over NVLink; ranks outside the range return at once. */
PP_API int pp_comm_all_gather_rows(pp_handle h, void* buf, const long long* rows_per_member, size_t row_bytes,
                                   int first_rank, int n_members, void* stream);

/* frames [T,3,H,W] in [-1,1]  ->  flows_f, flows_b [T-1,2,H,W].  fp16 activations, fp32 accumulation. */
PP_API int pp_raft_bidir(pp_handle h, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                  void* stream);
/* The same at fp32 accuracy (the node's fp16="disable"): fp32 activations, every convolution and the correlation as
 * error-compensated tf32 GEMMs (3xTF32), fp32 correlation pyramid.  Needs the RAFT weights also registered as split
 * images under "<name>.tf32" (engine.py registers both). */
PP_API int pp_raft_bidir_fp32(pp_handle h, const float* frames, int T, int H, int W, int iters, float* flows_f,
                              float* flows_b, void* stream);
/* flows [T-1,2,H,W], flow_masks [T,1,H,W]  ->  completed flows [T-1,2,H,W] (prediction inside the mask). */
PP_API int pp_flow_complete(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T, int H,
                     int W, float* out_f, float* out_b, void* stream);
/* The same call made collectively by the ranks [team_first, team_first + team_size) of the communicator on the same
 * (replicated) inputs; ranks outside the team return at once.  The two direction passes go to the two halves of the
 * team, the per-frame encoder / decoder is sharded inside a half (encoder with the +-8-frame temporal halo), the
 * serial recurrence runs on every rank of its half; NCCL all-gathers of the encoder features (inside a half) and of
 * the completed flows (whole team) leave the full result on every rank of the team.  team_size 1 = pp_flow_complete. */
PP_API int pp_flow_complete_dist(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T,
                                 int H, int W, float* out_f, float* out_b, int team_first, int team_size, void* stream);
/* pp_flow_complete / pp_flow_complete_dist at fp32 accuracy (the node's fp16="disable"): fp32 activations, every
 * convolution as an error-compensated tf32 GEMM (3xTF32), an fp32 deformable sampler and bilinear upsampling, and a
 * combine that returns the input flow unchanged outside the mask.  The propagation step runs one launch per layer, and
 * the per-frame decoder runs in frame batches sized to the free arena (the result does not depend on the batch size).
 * Needs the flow-completion weights also registered as split images under "<name>.tf32" (engine.py registers both). */
PP_API int pp_flow_complete_fp32(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T,
                                 int H, int W, float* out_f, float* out_b, void* stream);
PP_API int pp_flow_complete_dist_fp32(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks,
                                      int T, int H, int W, float* out_f, float* out_b, int team_first, int team_size,
                                      void* stream);
/* frames [T,3,H,W], masks [T,1,H,W], completed flows  ->  updated frames [T,3,H,W], updated masks [T,1,H,W]. */
PP_API int pp_image_propagate(pp_handle h, const float* frames, const float* masks, const float* flows_f,
                       const float* flows_b, int T, int H, int W, float* updated_frames, float* updated_masks,
                       void* stream);
/* The same at fp32 accuracy (the node's fp16="disable"): frames, masks and flows stay fp32 through the 2(T-1) steps,
 * and the bilinear weights and sums and the forward-backward test are rounded as torch evaluates them in fp32 on the
 * CPU, so the discrete decisions (fb validity, the 0.1 mask threshold, the nearest-pixel warp) are the ones the
 * reference takes there.  pp_image_propagate stores fp16 frames and flows. */
PP_API int pp_image_propagate_fp32(pp_handle h, const float* frames, const float* masks, const float* flows_f,
                                   const float* flows_b, int T, int H, int W, float* updated_frames,
                                   float* updated_masks, void* stream);
/* Generator session over one clip: encodes all T frames once. */
PP_API int pp_gen_begin(pp_handle h, const float* updated_frames, const float* masks_dilated, const float* updated_masks,
                 const float* flows_f, const float* flows_b, int T, int H, int W, void* stream);
/* Same, encoding only the frames with frames_needed[f] != 0 (host array of T bytes): a rank that runs a shard of the
 * sliding windows encodes the frames those windows touch; windows passed to pp_gen_run must stay inside that set. */
PP_API int pp_gen_begin_subset(pp_handle h, const float* updated_frames, const float* masks_dilated,
                               const float* updated_masks, const float* flows_f, const float* flows_b, int T, int H, int W,
                               const unsigned char* frames_needed, void* stream);
/* One sliding window: frame_ids[0..l_t) are consecutive local frames, frame_ids[l_t..t) reference frames
 * (host array).  pred is fp16 [l_t][H][W][4] (rgb in [-1,1] + 1 unused lane). */
PP_API int pp_gen_window(pp_handle h, const int* frame_ids, int t, int l_t, void* pred_f16, void* stream);
/* All sliding windows of the clip in one batched pass: frame_ids is the concatenation of every window's
 * [local..., reference...] ids, win_t / win_lt the per-window frame counts (host arrays).
 * pred is fp16 [sum(win_lt)][H][W][4] in window order. */
PP_API int pp_gen_run(pp_handle h, const int* frame_ids, const int* win_t, const int* win_lt, int n_windows,
                      void* pred_f16, void* stream);
PP_API int pp_gen_end(pp_handle h);
/* uint8 composite with the reference's truncation / 0.5-0.5 blending order.  frame_ids / first_visit are
 * device int32 arrays of length l_t; orig / comp are uint8 [T][H][W][3]; masks float32 [T,1,H,W].
 * half_math = 1 reproduces the roundings of the reference's fp16="enable" mode ((pred+1)/2 and *255 evaluated in
 * half precision before the uint8 truncation), 0 its fp32 mode. */
PP_API int pp_composite(pp_handle h, const void* pred_f16, const float* masks_dilated, const uint8_t* orig, uint8_t* comp,
                 const int* frame_ids_dev, const int* first_visit_dev, int l_t, int H, int W, int half_math,
                 void* stream);

/* Device pre-processing when no resize is needed (reference utils/image_utils.py:106-197): image [T,H,W,3]
 * float 0..1 -> uint8 (truncate) [T,H,W,3] + frames [T,3,H,W] in [-1,1]; mask [mask_frames,H,W] float ->
 * 8-bit -> cross dilation x N -> flow_masks / masks_dilated [T,1,H,W] in {0,1}.  All device pointers. */
PP_API int pp_preprocess(pp_handle h, const float* image, const float* mask, int mask_frames, int T, int H, int W,
                         int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8, float* frames, float* flow_masks,
                         float* masks_dilated, void* stream);
/* The same with a resize to the processing size out_w x out_h (reference utils/image_utils.py:98-103: PIL
 * Image.resize, bicubic, on the 8-bit frames and on the 8-bit mask images) done on the device, bit-identical to
 * Pillow's 8-bit resampler (two passes, 22-bit fixed-point coefficients).  Outputs have the processing size. */
PP_API int pp_preprocess_resize(pp_handle h, const float* image, const float* mask, int mask_frames, int T, int H, int W,
                                int out_h, int out_w, int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8,
                                float* frames, float* flow_masks, float* masks_dilated, void* stream);
/* The same from 8-bit inputs already on the device (image_u8 [T,H,W,3], mask_u8 [mask_frames,H,W]): what is left of the
 * pre-processing after the float -> uint8 truncation, which a host can do itself (pp_host_quantize_u8) to move 1/4 of the
 * bytes over PCIe.  out_h / out_w equal to H / W: no resize. */
PP_API int pp_preprocess_u8(pp_handle h, const uint8_t* image_u8, const uint8_t* mask_u8, int mask_frames, int T, int H,
                            int W, int out_h, int out_w, int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8,
                            float* frames, float* flow_masks, float* masks_dilated, void* stream);
/* HOST helper, no GPU work: dst[i] = (uint8)trunc(clip(src[i] * 255, 0, 255)) in float32, the reference's conversion
 * (utils/image_utils.py:106-114, 128-134), on `threads` host threads; src / dst are host pointers. */
PP_API int pp_host_quantize_u8(const float* src, uint8_t* dst, long long n, int threads);
/* The same conversion on the device, for an IMAGE that is already there: src float, dst uint8, n elements. */
PP_API int pp_quantize_u8(pp_handle h, const float* src, uint8_t* dst, long long n, void* stream);
/* Device pre-processing of the Outpaint node (reference utils/image_utils.py:98-116, 178-252: convert_image_to_frames,
 * extrapolation, prepare_frames_and_masks_for_outpaint) from 8-bit frames image_u8 [T,H,W,3]: resized to rw x rh
 * when that differs from W x H (PIL's 8-bit bicubic resampler, bit for bit, as in pp_preprocess_resize), placed at
 * (int((pw - rw) / 2), int((ph - rh) / 2)) on a zero pw x ph canvas -> orig_u8 [T,ph,pw,3], frames [T,3,ph,pw] in
 * [-1,1], and the band masks [T,1,ph,pw] in {0,1}: masks_dilated is 1 outside the frames, flow_masks is that band
 * plus a 4-px inset into the frames on each axis whose band is wider than 10 px.  Requires 0 < rw <= pw, 0 < rh <= ph.
 * All device pointers. */
PP_API int pp_preprocess_outpaint_u8(pp_handle h, const uint8_t* image_u8, int T, int H, int W, int rw, int rh, int pw,
                                     int ph, uint8_t* orig_u8, float* frames, float* flow_masks, float* masks_dilated,
                                     void* stream);
/* uint8 frames -> float32 / 255 (reference handle_output, utils/image_utils.py:276-290). */
PP_API int pp_postprocess(pp_handle h, const uint8_t* comp_u8, float* image_out, long long n, void* stream);

/* Kernels launched by this handle since creation (bench accounting), and the arena high-water mark. */
PP_API long long pp_launch_count(pp_handle h);
PP_API size_t pp_workspace_peak(pp_handle h);

/* Per-kernel timing with CUDA events on the launch stream (bench.py roofline): enable, run, dump a
 * tab-separated table "name count ms rows flops bytes" aggregated by kernel name. */
PP_API int pp_profile_enable(pp_handle h, int on);
PP_API int pp_profile_dump(pp_handle h, char* buf, size_t cap);

/* ---- single-operator entry points (unit tests and micro-benchmarks) ------------------------------------ */
/* Generic conv / linear through the wgmma implicit-GEMM kernel: x NHWC fp16 [N,H,W,cin_g*groups]. */
PP_API int pp_op_conv(pp_handle h, const char* name, const void* x_f16, int N, int H, int W, int stride, int pad, int dil,
               int replicate, int act, float slope, const void* residual_f16, void* out_f16, void* stream);
/* One stride-1 fp16 convolution into a channel slice: input x [N][H][W][x_C] from channel x_co (the layer's Cin, grouped
 * layers read and write their groups packed), zero padding ph x pw, output out [N][OH][OW][out_C] from channel out_co,
 * epilogue epi = 0: act2(act(acc + bias) * scale + aux0) with aux0 an optional residual [pix][aux0_C] at aux0_co;
 * epi = 1 (GRU z|r): z -> out, r * aux0 (h) -> aux1 (r*h); epi = 2 (GRU q): (1 - z) * h + z * tanh(acc + bias) -> out
 * with h = aux0, z = aux1. */
PP_API int pp_op_conv_ex(pp_handle h, const char* name, const void* x_f16, int x_C, int x_co, int N, int H, int W, int ph,
                         int pw, int epi, int act, float slope, float scale, int act2, const void* aux0_f16, int aux0_C,
                         int aux0_co, void* aux1_f16, int aux1_C, int aux1_co, void* out_f16, int out_C, int out_co,
                         void* stream);
/* One fp16 convolution of any layout a stage builds: nseg (1..6) input segments, segment i = channels
 * [x_co[i], x_co[i] + x_ch[i]) of x_f16[i] [N][H][W][x_C[i]], plus g * x_gstep[i] for group g; weights registered with
 * zero-padded input channels read the last segment zero-extended.  Stride sh x sw, padding ph x pw (zeros, or with
 * replicate the edge pixels), dilation dh x dw.  Output out [N][OH][OW][out_C] from channel out_co (+ g * out_gstep), fp16,
 * or with out_fp32 plain fp32.  Epilogue epi / act / slope / scale / act2 / aux0 / aux1 as in pp_op_conv_ex. */
PP_API int pp_op_conv_segs(pp_handle h, const char* name, int nseg, const void* const* x_f16, const int* x_C,
                           const int* x_co, const int* x_ch, const int* x_gstep, int N, int H, int W, int sh, int sw,
                           int ph, int pw, int dh, int dw, int replicate, int epi, int act, float slope, float scale,
                           int act2, const void* aux0_f16, int aux0_C, int aux0_co, void* aux1_f16, int aux1_C,
                           int aux1_co, void* out, int out_C, int out_co, int out_gstep, int out_fp32, void* stream);
/* The tile plan of the calling thread's last convolution launch, the first n of: kernel ('g' flat GEMM, 'h' halo tile,
 * 'i' implicit GEMM, 'p' recorded into a program, '?' none), MT (halo) or MB (gemm), N tile width, filter taps per weight
 * stage (halo), flat mode, TMA-store epilogue, patch / A stages, weight stages. */
PP_API int pp_op_conv_last_plan(int* plan, int n);
PP_API int pp_op_corr_lookup(pp_handle h, const void* l0, const void* l1, const void* l2, const void* l3,
                      const float* coords, void* out_f16, long long nq, int h8, int w8, void* stream);
/* Operators of the fp32 RAFT and flow-completion paths (pp_raft_bidir_fp32, pp_flow_complete_fp32).  Split tensors are fp32 [pix][hi C | lo C] with hi = tf32(x),
 * lo = x - hi; `*_C` is a tensor's channel count C, `*_co` / `*_ch` count channels.
 * One split-tf32 convolution with weights registered as a split image (Engine.register_conv_tf32): input x0 channels
 * [x0_co, x0_co + x0_ch) (then x1's, when x1 is not null), stride sh x sw, padding ph x pw (zeros, or with
 * replicate the edge pixels), dilation dh x dw, epilogue
 * epi = 0: act2(act(acc + bias) * scale + aux0), aux0 an optional split residual;
 * epi = 1 (GRU z|r): z -> out, r * aux0 (h) -> aux1 (r*h);  epi = 2 (GRU q): (1 - z) * h + z * tanh(acc + bias) -> out
 * with h = aux0, z = aux1.  out is split, written at channel out_co, or (out_fp32) plain fp32 [pix][out_C]. */
PP_API int pp_op_conv_tf32(pp_handle h, const char* name, const float* x0, int x0_C, int x0_co, int x0_ch, const float* x1,
                           int x1_C, int x1_co, int x1_ch, int N, int H, int W, int sh, int sw, int ph, int pw, int dh,
                           int dw, int replicate, int epi, int act, float slope, float scale, int act2, const float* aux0, int aux0_C, int aux0_co,
                           float* aux1, int aux1_C, int aux1_co, float* out, int out_C, int out_co, int out_fp32,
                           void* stream);
/* Modulated deformable sampling of pp_flow_complete_fp32 (3x3, pad 1, 16 offset groups): split inputs x0 [pix][hi C0 |
 * lo C0] and x1 [pix][hi C1 | lo C1] (C0 + C1 = 256, images of H x W), offs plain fp32 [pix][432] (raw offset-head output:
 * offsets max_mag * tanh, modulation sigmoid) -> split columns cols [pix][hi 2304 | lo 2304], K ordered (tap, channel).
 * x0, x1 and cols 16-byte aligned; x1 may be NULL when C1 = 0. */
PP_API int pp_op_dcn_sample_f32(pp_handle h, const float* x0, int C0, const float* x1, int C1, const float* offs, int N,
                                int H, int W, float max_mag, float* cols, void* stream);
/* Bilinear x2 upsampling (align_corners=True) of split tensors: src [N][H][W][hi C | lo C] -> dst [N][2H][2W][hi C | lo C]
 * (16-byte aligned, C a multiple of 4). */
PP_API int pp_op_upsample2x_f32(pp_handle h, const float* src, float* dst, int N, int H, int W, int C, void* stream);
/* InstanceNorm2d (eps 1e-5, no affine) of N images [HW][C] (+relu) (then relu(residual + .)): fp16 [pix][C] or, with
 * fp32, split tensors.  out may be x. */
PP_API int pp_op_instnorm(pp_handle h, const void* x, const void* residual, void* out, int N, int HW, int C, int relu,
                          int fp32, void* stream);
/* RAFT correlation pyramid of `pairs` frame pairs: fmap1 / fmap2 [pairs][h8*w8][256] (fp16, or with fp32 split) ->
 * levels l0..l3 [pairs*h8*w8][(h8 >> l) * (w8 >> l)] (fp16 / fp32). */
PP_API int pp_op_corr_pyramid(pp_handle h, const void* fmap1, const void* fmap2, int pairs, int h8, int w8, int fp32,
                              void* l0, void* l1, void* l2, void* l3, void* stream);
/* pp_op_corr_lookup on an fp32 pyramid: out is split [nq][hi 352 | lo 352] (channels 324..351 zero). */
PP_API int pp_op_corr_lookup_f32(pp_handle h, const float* l0, const float* l1, const float* l2, const float* l3,
                                 const float* coords, float* out, long long nq, int h8, int w8, void* stream);
/* RAFT convex 8x upsampling: coords1 [B*h8*w8][2], mask [B*h8*w8][576] fp16 (or with fp32 split) -> out [B][2][8h8][8w8]. */
PP_API int pp_op_convex_upsample(pp_handle h, const float* coords1, const void* mask, float* out, int B, int h8, int w8,
                                 int fp32, void* stream);
PP_API int pp_op_imgprop_step(pp_handle h, const void* cur4_f16, const void* prop_in4_f16, void* prop_out4_f16,
                       const void* flow_prop_f16, const void* flow_check_f16, int H, int W, void* stream);
/* One image-propagation step of pp_image_propagate_fp32: pixels float32 [H][W][4] (r, g, b, mask), flows float32
 * [H][W][2]. */
PP_API int pp_op_imgprop_step_f32(pp_handle h, const float* cur4, const float* prop_in4, float* prop_out4,
                                  const float* flow_prop, const float* flow_check, int H, int W, void* stream);
/* Operators of the generator (pp_gen_run), fp16 NHWC, each one launch of the kernel the stage runs.  Token grids: gh x gw
 * tokens of a frame (unfold 7x7, stride 3, pad 3 of an h4 x w4 feature map), padded to nh x nw (multiples of 5 x 9).
 * Sparse window attention of sliding windows whose frames are concatenated (window w owns win_t[w] >= 2 frames, host
 * array): qkv [frames][nh*nw][q 512 | k 512 | v 512], pooled pkv [frames][n_pool][k 512 | v 512] -> out [frames][gh][gw][512];
 * win_flags_dev [n_windows][(nh/5)*(nw/9)] (device) selects the masked 5x9 windows; key frames are parity, parity+2, ... */
PP_API int pp_op_attention(pp_handle h, const void* qkv_f16, const void* pkv_f16, void* out_f16, const int* win_flags_dev,
                           const int* win_t, int n_windows, int gh, int gw, int n_pool, int parity, void* stream);
/* LayerNorm over 512 channels (eps 1e-5, fp32 gamma / beta): x [t*gh*gw][512] -> out [t][nh][nw][512]; rows of the
 * padding are not written. */
PP_API int pp_op_layernorm(pp_handle h, const void* x_f16, const float* gamma, const float* beta, void* out_f16, int t,
                           int gh, int gw, int nh, int nw, void* stream);
/* Depthwise 4x4 stride-4 pooling: x [t][nh][nw][C], w fp32 [16 taps][C], b fp32 [C] -> out [t][ph][pw][C] with
 * ph = (nh - 4) / 4 + 1, pw = (nw - 4) / 4 + 1. */
PP_API int pp_op_pool_tokens(pp_handle h, const void* x_f16, const float* w, const float* b, void* out_f16, int t, int nh,
                             int nw, int C, void* stream);
/* Masked-window flags: mask4 [frames][h4][w4][cs] (channel co), sliding window w covers frames win_f0[w] ..
 * win_f0[w] + win_lt[w] - 1 (host arrays) -> flags_dev [n_windows][(nh/5)*(nw/9)] (device int32). */
PP_API int pp_op_window_flags(pp_handle h, const void* mask4_f16, int cs, int co, const int* win_f0, const int* win_lt,
                              int n_windows, int h4, int w4, int* flags_dev, void* stream);
/* F.fold(7x7, stride 3, pad 3) of x [t*gh*gw][cs] (column (ky*7 + kx)*C + c) -> out [t][H][W][C]; gh / gw derived from
 * H / W; normalise divides by the overlap count, gelu applies erf-GELU after it. */
PP_API int pp_op_fold(pp_handle h, const void* x_f16, int cs, void* out_f16, int t, int H, int W, int C, int normalise,
                      int gelu, void* stream);
/* DCN condition of one feature-propagation step: cur / prop [N][H][W][128], flows [N][H][W][2], mask2 [N][H][W][8] ->
 * cond [N][H][W][264] = (cur 128 | prop warped by flow_prop 128 | flow_prop 2 | fb validity 1 | mask2[0..1] 2 | 0 0 0). */
PP_API int pp_op_featprop_cond(pp_handle h, const void* cur_f16, const void* prop_f16, const void* flow_prop_f16,
                               const void* flow_check_f16, const void* mask2_f16, void* cond_f16, int N, int H, int W,
                               void* stream);
/* fp16 modulated deformable sampling (3x3, pad 1, 16 offset groups of (C0 + C1) / 16 channels, C0 + C1 = 128 or 256):
 * x0 [pix][x0_cs] channels 0..C0-1, x1 [pix][x1_cs] channels 0..C1-1 (x1 may be NULL when C1 = 0), offs [pix][432];
 * offsets max_mag * tanh, plus, with flow not NULL, the flow (x at channel flow_co, y at flow_co + 1 of [pix][flow_cs]);
 * -> cols [pix][9 * (C0 + C1)] ordered (tap, channel). */
PP_API int pp_op_dcn_sample(pp_handle h, const void* x0_f16, int x0_cs, int C0, const void* x1_f16, int x1_cs, int C1,
                            const void* offs_f16, const void* flow_f16, int flow_cs, int flow_co, float max_mag,
                            void* cols_f16, int N, int H, int W, void* stream);
/* 1/4 downsampling of pp_gen_begin: flows fp32 [n_flows][2][H][W] -> bilinear / 4 [n_flows][H/4][W/4][2]; masks fp32
 * [n_masks][1][H][W] -> nearest, channel mask_co of [n_masks][H/4][W/4][8].  Either pair may be NULL. */
PP_API int pp_op_downsample4(pp_handle h, const float* flows, void* flows4_f16, int n_flows, const float* masks,
                             void* masks4_f16, int mask_co, int n_masks, int H, int W, void* stream);
/* Bilinear x2 upsampling (align_corners=True): src [N][H][W][C] -> dst [N][2H][2W][C] (C a multiple of 8). */
PP_API int pp_op_upsample2x(pp_handle h, const void* src_f16, void* dst_f16, int N, int H, int W, int C, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PROPAINTER_B200_H */

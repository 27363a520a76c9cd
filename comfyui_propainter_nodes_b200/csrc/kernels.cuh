// Launchers of the hand-written HBM-bound kernels (everything that is not a tensor-core contraction)
// plus the window attention.  Activations are NHWC fp16 unless a name says otherwise;
// `cs` = channel stride (elements per pixel), `co` = channel offset inside the pixel.
// A launcher that serves both storage precisions has one name, overloaded or templated on the element type of its
// tensors.  __half: fp16 [pix][C].  float: in RAFT a split-tf32 pair tensor [pix][hi C | lo C] (conv_igemm.cuh) given
// by its real channel count C, and a plain fp32 correlation pyramid; in image propagation float4 pixels, float2 flows.
#pragma once
#include "pp_common.cuh"

// ---- layout / elementwise (kernels_basic.cu) ---------------------------------------------------
// frames [N][C][H][W] fp32 -> a stage's activation layout, `cs` channels per pixel, channels C..cs-1 zero (the fp32
// form is in kernels_raft.cu).  fp16 only: the C channels go to the slice starting at dst_co, of which channels
// C..zero_fill_to-1 are zero-filled (< 0: to the end of the pixel).
int pp_k_nchw_to_act(const float* src, __half* dst, int N, int C, int H, int W, int cs, cudaStream_t st, int dst_co = 0,
                     int zero_fill_to = -1);
int pp_k_nchw_to_act(const float* src, float* dst, int N, int C, int H, int W, int cs, cudaStream_t st);
int pp_k_upsample2x(const __half* src, int src_cs, int src_co, __half* dst, int dst_cs, int dst_co, int N, int H,
                    int W, int C, cudaStream_t st);
// split-tf32 form: src [N][H][W][hi C | lo C] -> dst [N][2H][2W][hi C | lo C]
int pp_k_upsample2x(const float* src, float* dst, int N, int H, int W, int C, cudaStream_t st);
int pp_k_gather_blocks(void* dst, const void* src, const int* idx_dev, long long n, long long block_bytes,
                       cudaStream_t st);
int pp_k_copy_blocks(void* dst, const int* dst_idx_dev, const void* src, const int* src_idx_dev, long long n,
                     long long block_bytes, cudaStream_t st);

// ---- RAFT (kernels_raft.cu) ---------------------------------------------------------------------
size_t pp_k_instnorm_scratch_floats(int N, int HW, int C);
// sums: scratch of pp_k_instnorm_scratch_floats floats; leaves [N][sum x | sum x^2] (fp16) or [N][mean | variance] (fp32)
template <class E>
int pp_k_instnorm_stats(const E* x, int N, int HW, int C, float* sums, cudaStream_t st);
template <class E>
int pp_k_instnorm_apply(const E* x, const float* sums, const E* residual, E* out, int N, int HW, int C, int relu,
                        cudaStream_t st);
int pp_k_pack_b_operand(const __half* src /*[G][R][K]*/, __half* dst, int G, int R, int R_pad, int K, cudaStream_t st);
int pp_k_pack_b_operand(const float* src /*[G][R][hi K | lo K]*/, float* dst, int G, int R, int R_pad, int K,
                        cudaStream_t st);
template <class E>
int pp_k_corr_pool(const E* src, E* dst, long long nq, int h, int w, cudaStream_t st);
template <class E>
int pp_k_corr_lookup(const E* l0, const E* l1, const E* l2, const E* l3, const float* coords, E* out, int out_C,
                     long long nq, int h8, int w8, cudaStream_t st);
int pp_k_cnet_split(const __half* c, __half* hx, int hx_C, long long npix, cudaStream_t st);
int pp_k_cnet_split(const float* c, float* hx, int hx_C, long long npix, cudaStream_t st);
// coords1 = coords0 (delta == nullptr) or coords1 + delta; the flow goes to channels hx_flow_co, +1 of the GRU state
// and, fp16, to flow8 [.][8] for the 7x7 patches (fp32 takes them from coords1)
int pp_k_raft_coords(const float* delta, float* coords1, __half* flow8, __half* hx, int hx_C, int hx_flow_co, int B,
                     int h8, int w8, cudaStream_t st);
int pp_k_raft_coords(const float* delta, float* coords1, float* hx, int hx_C, int hx_flow_co, int B, int h8, int w8,
                     cudaStream_t st);
int pp_k_flow_patch7x7(const __half* flow8, __half* out /*[M][128]*/, int B, int h8, int w8, cudaStream_t st);
int pp_k_flow_patch7x7(const float* coords1, float* out /*[M][hi 128 | lo 128]*/, int B, int h8, int w8,
                       cudaStream_t st);
template <class E>
int pp_k_convex_upsample(const float* coords1, const E* mask, float* out_nchw, int B, int h8, int w8, cudaStream_t st);

// ---- propagation (kernels_prop.cu) --------------------------------------------------------------
// image propagation, E = __half: pixels 4 x fp16 (r, g, b, mask), flows __half2; E = float: float4 / float2 with fp32
// sums in PyTorch's order
template <class E>
int pp_k_imgprop_step(const E* cur, const E* prop_in, E* prop_out, const E* flow_prop, const E* flow_check, int H,
                      int W, cudaStream_t st);
// bwd / fwd must hold copies of in4; scratch = 8 ints (bbox[4], barrier counter, pad)
template <class E>
int pp_k_imgprop_run(const E* in4, E* bwd, E* fwd, const E* ff, const E* fbk, const float* masks, int T, int H, int W,
                     int* scratch, cudaStream_t st);
template <class E>
int pp_k_imgprop_pack(const float* frames, const float* masks, E* dst, int T, int H, int W, cudaStream_t st);
template <class E>
int pp_k_imgprop_finish(const E* prop, const float* frames, const float* masks, float* upd_frames, float* upd_masks,
                        int T, int H, int W, cudaStream_t st);
template <class E>
int pp_k_flow_to_nhwc2(const float* src, E* dst, int n, int H, int W, cudaStream_t st);
int pp_k_rfc_pack_input(const float* flows, const float* masks, __half* dst, long long dst_tstride_pix, int T, int H,
                        int W, int reverse_time, cudaStream_t st);
int pp_k_rfc_combine(const __half* pred, int pred_cs, long long pred_tstride_pix, const float* gt, const float* masks,
                     float* out, int T, int H, int W, int reverse_time, cudaStream_t st);
int pp_k_dcn_sample(const __half* x0, int x0_cs, int x0_co, int C0, const __half* x1, int x1_cs, int x1_co, int C1,
                    const __half* offs, int offs_cs, const __half* flow, int flow_cs, int flow_co, float max_mag,
                    __half* cols, int N, int H, int W, cudaStream_t st);
// flow completion, fp32 (split-tf32 activations): input [T][hi 4 | lo 4] (flow * (1 - m), m, 0), plain fp32 pred, and
// the deformable sampler on split x0 / x1 (C0 + C1 = 256) with plain fp32 offsets -> split columns [pix][hi 9C | lo 9C]
int pp_k_rfc_pack_input(const float* flows, const float* masks, float* dst, long long dst_tstride_pix, int T, int H,
                        int W, int reverse_time, cudaStream_t st);
int pp_k_rfc_combine(const float* pred, int pred_cs, long long pred_tstride_pix, const float* gt, const float* masks,
                     float* out, int T, int H, int W, int reverse_time, cudaStream_t st);
int pp_k_dcn_sample(const float* x0, int C0, const float* x1, int C1, const float* offs, int offs_cs, float max_mag,
                    float* cols, int N, int H, int W, cudaStream_t st);
int pp_k_featprop_cond(const __half* cur, int cur_cs, const __half* prop, int prop_cs, const __half* flow_prop,
                       const __half* flow_check, const __half* mask2, int mask_cs, __half* cond, int cond_cs, int N,
                       int H, int W, int C, cudaStream_t st);
int pp_k_downsample_flow4(const float* flow, __half* dst, int n, int H, int W, cudaStream_t st);
int pp_k_downsample_mask4(const float* m, __half* dst, int dst_cs, int dst_co, int n, int H, int W, cudaStream_t st);

// ---- transformer (kernels_xfmr.cu, attention.cu) ------------------------------------------------
int pp_k_layernorm(const __half* x, const float* gamma, const float* beta, __half* out, long long rows, int gh, int gw,
                   int nh, int nw, cudaStream_t st);
int pp_k_pool_tokens(const __half* x, const float* w, const float* b, __half* out, int t, int nh, int nw, int ph,
                     int pw, int C, cudaStream_t st);
int pp_k_window_flags(const __half* mask4, int cs, int co, const int* win_f0, const int* win_lt, int n_windows, int h4,
                      int w4, int gh, int gw, int nwh, int nww, int* flags, cudaStream_t st);
int pp_k_fold(const __half* x, int cs, __half* out, int t, int H, int W, int C, int gh, int gw, int normalise,
              int gelu, cudaStream_t st);
int pp_k_attention(const __half* q, const __half* k, const __half* v, int qkv_cs, const __half* pk, const __half* pv,
                   int pool_cs, __half* out, int out_cs, const int* win_flags, const int* ring_idx,
                   const int* sw_frame_off, const int* sw_t, int n_sliding, int t_max, int gh, int gw, int nh, int nw,
                   int n_pool, int t_parity, int* key_tab, int key_tab_stride, cudaStream_t st);
int pp_k_composite(const __half* pred, int pred_cs, const float* masks, const uint8_t* orig, uint8_t* comp,
                   const int* frame_ids, const int* first_visit, int lt, int H, int W, int half_math, cudaStream_t st);

// ---- device pre/post-processing (kernels_pre.cu) --------------------------------------------------
int pp_k_quantize_frames(const float* img, uint8_t* u8, float* frames, int T, int H, int W, cudaStream_t st);
int pp_k_prepare_masks(const float* mask, int Tm, int T, int H, int W, int iters_flow, int iters_dil, uint8_t* scratch,
                       float* flow_masks, float* masks_dilated, cudaStream_t st);
int pp_k_u8_to_unit_float(const uint8_t* src, float* dst, long long n, cudaStream_t st);
int pp_k_resize_bicubic_u8(const uint8_t* src, uint8_t* dst, uint8_t* tmp, int* coef, size_t coef_ints, int T, int H, int W,
                           int C, int OH, int OW, cudaStream_t st);
int pp_k_quantize_u8(const float* img, uint8_t* u8, long long n, cudaStream_t st);
int pp_k_u8_to_frames(const uint8_t* u8, float* frames, int T, int H, int W, cudaStream_t st);
int pp_k_dilate_masks_u8(const uint8_t* mask_u8, int Tm, int T, int H, int W, int iters_flow, int iters_dil,
                         float* flow_masks, float* masks_dilated, cudaStream_t st);
int pp_k_outpaint_canvas(const uint8_t* window, int T, int rw, int rh, int pw, int ph, uint8_t* orig, float* frames,
                         float* flow_masks, float* masks_dilated, cudaStream_t st);

// Launchers of the hand-written HBM-bound kernels (everything that is not a tensor-core contraction)
// plus the window attention.  Activations are NHWC fp16 unless a name says otherwise;
// `cs` = channel stride (elements per pixel), `co` = channel offset inside the pixel.
#pragma once
#include "pp_common.cuh"

// ---- layout / elementwise (kernels_basic.cu) ---------------------------------------------------
int pp_k_nchw_f32_to_nhwc_f16(const float* src, __half* dst, int N, int C, int H, int W, int dst_cs, int dst_co,
                              int zero_fill_to, cudaStream_t st);
int pp_k_nhwc_f16_to_nchw_f32(const __half* src, int src_cs, int src_co, float* dst, int N, int C, int H, int W,
                              cudaStream_t st);
int pp_k_upsample2x(const __half* src, int src_cs, int src_co, __half* dst, int dst_cs, int dst_co, int N, int H,
                    int W, int C, cudaStream_t st);
int pp_k_copy_channels(const __half* src, int src_cs, int src_co, __half* dst, int dst_cs, int dst_co, long long npix,
                       int C, cudaStream_t st);
int pp_k_fill_f16(__half* dst, long long n, float v, cudaStream_t st);
int pp_k_gather_blocks(void* dst, const void* src, const int* idx_dev, long long n, long long block_bytes,
                       cudaStream_t st);
int pp_k_copy_blocks(void* dst, const int* dst_idx_dev, const void* src, const int* src_idx_dev, long long n,
                     long long block_bytes, cudaStream_t st);

// ---- RAFT (kernels_raft.cu) ---------------------------------------------------------------------
size_t pp_k_instnorm_scratch_floats(int N, int HW, int C);
int pp_k_instnorm_stats(const __half* x, int N, int HW, int C, float* sums /*[N][2][C]*/, cudaStream_t st);
int pp_k_instnorm_apply(const __half* x, const float* sums, const __half* residual, __half* out, int N, int HW, int C,
                        int relu, cudaStream_t st);
int pp_k_pack_b_operand(const __half* src /*[G][R][K]*/, __half* dst, int G, int R, int R_pad, int K, cudaStream_t st);
int pp_k_corr_pool(const __half* src, __half* dst, long long nq, int h, int w, cudaStream_t st);
int pp_k_corr_lookup(const __half* l0, const __half* l1, const __half* l2, const __half* l3, const float* coords,
                     __half* out, int out_cs, long long nq, int P, int h8, int w8, cudaStream_t st);
int pp_k_cnet_split(const __half* c, __half* hx, int hx_cs, long long npix, cudaStream_t st);
int pp_k_raft_coords_init(float* coords1, __half* flow8, __half* hx, int hx_cs, int hx_flow_co, int B, int h8, int w8,
                          cudaStream_t st);
int pp_k_raft_coords_update(const float* delta, float* coords1, __half* flow8, __half* hx, int hx_cs, int hx_flow_co,
                            int B, int h8, int w8, cudaStream_t st);
int pp_k_flow_patch7x7(const __half* flow8, __half* out /*[M][128]*/, int B, int h8, int w8, cudaStream_t st);
int pp_k_convex_upsample(const float* coords1, const __half* mask, float* out_nchw, int B, int h8, int w8,
                         cudaStream_t st);
// fp32 RAFT path: split-tf32 pair tensors [pix][hi C | lo C] (conv_igemm.cuh), fp32 correlation pyramid
int pp_k_nchw_f32_to_split(const float* src, float* dst, int N, int C, int H, int W, int cs, cudaStream_t st);
int pp_k_instnorm_stats_f32(const float* x, int N, int HW, int C, float* sums /*[N][mean C | variance C]*/,
                            cudaStream_t st);
int pp_k_instnorm_apply_f32(const float* x, const float* sums, const float* residual, float* out, int N, int HW, int C,
                            int relu, cudaStream_t st);
int pp_k_pack_b_operand_split(const float* src, float* dst, int G, int R, int R_pad, int K, cudaStream_t st);
int pp_k_corr_pool_f32(const float* src, float* dst, long long nq, int h, int w, cudaStream_t st);
int pp_k_corr_lookup_f32(const float* l0, const float* l1, const float* l2, const float* l3, const float* coords,
                         float* out /*[nq][hi out_C | lo out_C]*/, int out_C, long long nq, int h8, int w8, cudaStream_t st);
int pp_k_cnet_split_f32(const float* c, float* hx, int hx_C, long long npix, cudaStream_t st);
// delta == nullptr: coords1 = coords0 (init)
int pp_k_raft_coords_f32(const float* delta, float* coords1, float* hx, int hx_C, int hx_flow_co, int B, int h8, int w8,
                         cudaStream_t st);
int pp_k_flow_patch7x7_f32(const float* coords1, float* out /*[M][hi 128 | lo 128]*/, int B, int h8, int w8, cudaStream_t st);
int pp_k_convex_upsample_f32(const float* coords1, const float* mask, float* out_nchw, int B, int h8, int w8,
                             cudaStream_t st);

// ---- propagation (kernels_prop.cu) --------------------------------------------------------------
int pp_k_imgprop_step(const __half* cur, const __half* prop_in, __half* prop_out, const __half* flow_prop,
                      const __half* flow_check, int H, int W, cudaStream_t st);
int pp_k_imgprop_run(const __half* in4, __half* bwd, __half* fwd, const __half* ff, const __half* fbk,
                     const float* masks, int T, int H, int W, int* scratch, cudaStream_t st);
int pp_k_imgprop_pack(const float* frames, const float* masks, __half* dst, int T, int H, int W, cudaStream_t st);
int pp_k_imgprop_finish(const __half* prop, const float* frames, const float* masks, float* upd_frames,
                        float* upd_masks, int T, int H, int W, cudaStream_t st);
int pp_k_flow_to_nhwc2(const float* src, __half* dst, int n, int H, int W, cudaStream_t st);
// fp32 image propagation: pixels float4 (r, g, b, mask), flows float2, fp32 sums in PyTorch's order
int pp_k_imgprop_step_f32(const float* cur, const float* prop_in, float* prop_out, const float* flow_prop,
                          const float* flow_check, int H, int W, cudaStream_t st);
int pp_k_imgprop_run_f32(const float* in4, float* bwd, float* fwd, const float* ff, const float* fbk,
                         const float* masks, int T, int H, int W, int* scratch, cudaStream_t st);
int pp_k_imgprop_pack_f32(const float* frames, const float* masks, float* dst, int T, int H, int W, cudaStream_t st);
int pp_k_imgprop_finish_f32(const float* prop, const float* frames, const float* masks, float* upd_frames,
                            float* upd_masks, int T, int H, int W, cudaStream_t st);
int pp_k_flow_to_nhwc2_f32(const float* src, float* dst, int n, int H, int W, cudaStream_t st);
int pp_k_rfc_pack_input(const float* flows, const float* masks, __half* dst, long long dst_tstride_pix, int T, int H,
                        int W, int reverse_time, cudaStream_t st);
int pp_k_rfc_combine(const __half* pred, int pred_cs, long long pred_tstride_pix, const float* gt, const float* masks,
                     float* out, int T, int H, int W, int reverse_time, cudaStream_t st);
int pp_k_dcn_sample(const __half* x0, int x0_cs, int x0_co, int C0, const __half* x1, int x1_cs, int x1_co, int C1,
                    const __half* offs, int offs_cs, const __half* flow, int flow_cs, int flow_co, float max_mag,
                    __half* cols, int N, int H, int W, cudaStream_t st);
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



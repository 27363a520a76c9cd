// extern "C" surface of libpropainter_b200.so (declared in include/propainter_b200.h).
#include <math.h>
#include <string.h>

#include <thread>
#include <vector>

#include "../../include/propainter_b200.h"
#include "engine.cuh"

// Makes the engine's device current for the duration of one API call and restores the caller's device afterwards.
struct DeviceGuard {
  int prev = -1;
  bool changed = false, ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) {
      ok = cudaSetDevice(dev) == cudaSuccess;
      changed = ok;
    }
  }
  ~DeviceGuard() {
    if (changed && prev >= 0) cudaSetDevice(prev);
  }
};

#define PP_HANDLE(h)                                     \
  if ((h) == nullptr) {                                  \
    pp_set_error("null engine handle");                  \
    return PP_ERR_ARG;                                   \
  }                                                      \
  PPEngine& e = *reinterpret_cast<PPEngine*>(h);         \
  DeviceGuard _dev_guard(e.device);                      \
  if (!_dev_guard.ok) {                                  \
    pp_set_error("cudaSetDevice(%d) failed", e.device);  \
    return PP_ERR_CUDA;                                  \
  }

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
// null counts as aligned: optional tensors are checked only when given
static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Restores the arena to its state at entry on EVERY exit of a stage call (error paths included): a failed call
// ("workspace exhausted", bad argument after a partial allocation) must not shrink the workspace of the cached engine.
struct ArenaGuard {
  PPArena& a;
  size_t m;
  bool keep = false;
  explicit ArenaGuard(PPArena& arena) : a(arena), m(arena.mark()) {}
  ~ArenaGuard() { if (!keep) a.release(m); }
};

// pp_op_instnorm / pp_op_corr_pyramid take tensors of either precision as void* plus an fp32 flag: E is the element type
template <class E>
static int op_instnorm(PPEngine& e, const void* x, const void* residual, void* out, int N, int HW, int C, int relu,
                       cudaStream_t st) {
  ArenaGuard guard(e.arena);
  float* sums;
  PP_TRY(pp_alloc(e, &sums, pp_k_instnorm_scratch_floats(N, HW, C), "instnorm sums"));
  PP_TRY(pp_k_instnorm_stats(static_cast<const E*>(x), N, HW, C, sums, st));
  PP_TRY(pp_k_instnorm_apply(static_cast<const E*>(x), sums, static_cast<const E*>(residual), static_cast<E*>(out), N,
                             HW, C, relu, st));
  PP_CUDA_CHECK(cudaStreamSynchronize(st));   // the scratch goes back to the arena on return
  return PP_OK;
}

template <class E>
static int op_corr_pyramid(PPEngine& e, const void* fmap1, const void* fmap2, int pairs, int h8, int w8, void* l0,
                           void* l1, void* l2, void* l3, cudaStream_t st) {
  ArenaGuard guard(e.arena);
  const int P = h8 * w8, P_pad = pp_raft_corr_pad(P);
  E* fpack;   // 256 values per row, fp32: the three segments [hi; hi; lo]
  PP_TRY(pp_alloc(e, &fpack, (size_t)pairs * P_pad * 256 * (sizeof(E) == 4 ? 3 : 1), "fmap packed"));
  PP_TRY(pp_k_pack_b_operand(static_cast<const E*>(fmap2), fpack, pairs, P, P_pad, 256, st));
  e.launches++;
  E* const corr[4] = {static_cast<E*>(l0), static_cast<E*>(l1), static_cast<E*>(l2), static_cast<E*>(l3)};
  PP_TRY(pp_raft_corr_volume<E>(e, static_cast<const E*>(fmap1), fpack, pairs, P, P_pad, corr[0], st));
  PP_TRY(pp_raft_corr_pool(e, corr, (long long)pairs * P, h8, w8, st));
  PP_CUDA_CHECK(cudaStreamSynchronize(st));
  return PP_OK;
}

// pp_flow_complete_dist / _fp32: E is the element type of the stage
template <class E>
static int flow_complete_dist(pp_handle h, const char* what, const float* flows_f, const float* flows_b,
                              const float* flow_masks, int T, int H, int W, float* out_f, float* out_b, int team_first,
                              int team_size, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(flows_f && flows_b && flow_masks && out_f && out_b, "%s: null pointer", what);
  PP_REQUIRE(e.comm != nullptr || team_size <= 1, "%s: pp_comm_init was not called", what);
  PP_REQUIRE(team_first >= 0 && team_size >= 1 && team_first + team_size <= e.world,
             "%s: team [%d, %d) of %d ranks", what, team_first, team_first + team_size, e.world);
  ArenaGuard guard(e.arena);
  return pp_stage_flow_complete<E>(e, flows_f, flows_b, flow_masks, T, H, W, out_f, out_b, team_first, team_size,
                                   as_stream(stream));
}

extern "C" {

const char* pp_version(void) { return "propainter_b200 1 sm_90a"; }

int pp_create(int device, void* workspace, size_t workspace_bytes, pp_handle* out) {
  PP_REQUIRE(out != nullptr, "pp_create: out is null");
  PP_REQUIRE(workspace != nullptr && workspace_bytes >= (64u << 20), "pp_create: workspace must be >= 64 MiB");
  PP_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "pp_create: workspace must be 256-byte aligned");
  PP_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  PP_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  PP_REQUIRE(prop.major == 9 && prop.minor == 0, "pp_create: this library is built for sm_90a (Hopper H100); device %d is sm_%d%d",
             device, prop.major, prop.minor);
  PPEngine* e = new PPEngine();
  e->device = device;
  e->arena.base = static_cast<uint8_t*>(workspace);
  e->arena.cap = workspace_bytes;
  if (cudaMalloc(&e->prog_counter, 256) != cudaSuccess || cudaMemset(e->prog_counter, 0, 256) != cudaSuccess) {
    delete e;
    pp_set_error("pp_create: cudaMalloc of the program barrier word failed");
    return PP_ERR_CUDA;
  }
  *out = reinterpret_cast<pp_handle>(e);
  return PP_OK;
}

int pp_set_workspace(pp_handle h, void* workspace, size_t workspace_bytes) {
  PP_HANDLE(h);
  PP_REQUIRE(!e.gen.active, "pp_set_workspace: a generator session is active (call pp_gen_end first)");
  PP_REQUIRE(e.arena.off == 0, "pp_set_workspace: the arena is in use");
  PP_REQUIRE(workspace != nullptr && workspace_bytes >= (64u << 20), "pp_set_workspace: workspace must be >= 64 MiB");
  PP_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "pp_set_workspace: workspace must be 256-byte aligned");
  e.arena.base = static_cast<uint8_t*>(workspace);
  e.arena.cap = workspace_bytes;
  e.arena.peak = 0;
  return PP_OK;
}

int pp_destroy(pp_handle h) {
  if (h != nullptr) {
    PPEngine* e = reinterpret_cast<PPEngine*>(h);
    pp_comm_destroy_impl(*e);
    if (e->prog_counter != nullptr) cudaFree(e->prog_counter);
    delete e;
  }
  return PP_OK;
}

int pp_comm_unique_id(void* out128) {
  PP_REQUIRE(out128 != nullptr, "pp_comm_unique_id: null pointer");
  return pp_comm_unique_id_impl(out128);
}

int pp_comm_init(pp_handle h, const void* unique_id128, int rank, int world) {
  PP_HANDLE(h);
  PP_REQUIRE(unique_id128 != nullptr, "pp_comm_init: null id");
  return pp_comm_init_impl(e, unique_id128, rank, world);
}

int pp_comm_destroy(pp_handle h) {
  PP_HANDLE(h);
  return pp_comm_destroy_impl(e);
}

int pp_comm_all_gather_rows(pp_handle h, void* buf, const long long* rows_per_member, size_t row_bytes, int first_rank,
                            int n_members, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(buf != nullptr && rows_per_member != nullptr && row_bytes > 0 && n_members >= 1,
             "pp_comm_all_gather_rows: bad argument");
  std::vector<long long> off(n_members, 0);
  for (int m = 1; m < n_members; ++m) off[m] = off[m - 1] + rows_per_member[m - 1];
  return pp_comm_all_gather_blocks_impl(e, buf, off.data(), rows_per_member, row_bytes, first_rank, n_members,
                                        as_stream(stream));
}

int pp_register_conv(pp_handle h, const char* name, const void* w, const float* bias, int cout_g, int cout_g_pad,
                     int bn, int cin_g, int kh, int kw, int groups) {
  PP_HANDLE(h);
  PP_REQUIRE(name != nullptr && w != nullptr, "pp_register_conv: null argument");
  PP_REQUIRE(bn % 16 == 0 && bn >= 16 && bn <= 256 && cout_g_pad % bn == 0 && cout_g <= cout_g_pad && cin_g % 8 == 0,
             "pp_register_conv(%s): invalid packing (cout_g=%d pad=%d bn=%d cin_g=%d)", name, cout_g, cout_g_pad, bn,
             cin_g);
  PPPackedConv c;
  c.w = static_cast<const __half*>(w); c.b = bias;
  c.cout_g = cout_g; c.cout_g_pad = cout_g_pad; c.bn = bn; c.cin_g = cin_g; c.kh = kh; c.kw = kw; c.groups = groups;
  e.convs[name] = c;
  return PP_OK;
}

int pp_set_conv_macs(pp_handle h, const char* name, double macs_per_pixel) {
  PP_HANDLE(h);
  PP_REQUIRE(name != nullptr, "pp_set_conv_macs: null name");
  auto it = e.convs.find(name);
  PP_REQUIRE(it != e.convs.end(), "pp_set_conv_macs: conv '%s' is not registered", name);
  it->second.macs_per_pixel = macs_per_pixel;
  return PP_OK;
}

int pp_register_tensor(pp_handle h, const char* name, const void* ptr, size_t bytes) {
  PP_HANDLE(h);
  PP_REQUIRE(name != nullptr && ptr != nullptr, "pp_register_tensor: null argument");
  PPTensor t;
  t.ptr = ptr; t.bytes = bytes;
  e.tensors[name] = t;
  return PP_OK;
}

int pp_raft_bidir(pp_handle h, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                  void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(frames && flows_f && flows_b, "pp_raft_bidir: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_raft<__half>(e, frames, T, H, W, iters, flows_f, flows_b, as_stream(stream));
}

int pp_raft_bidir_fp32(pp_handle h, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                       void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(frames && flows_f && flows_b, "pp_raft_bidir_fp32: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_raft<float>(e, frames, T, H, W, iters, flows_f, flows_b, as_stream(stream));
}

int pp_flow_complete(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T, int H,
                     int W, float* out_f, float* out_b, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(flows_f && flows_b && flow_masks && out_f && out_b, "pp_flow_complete: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_flow_complete<__half>(e, flows_f, flows_b, flow_masks, T, H, W, out_f, out_b, 0, 1,
                                        as_stream(stream));
}

int pp_flow_complete_fp32(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T, int H,
                          int W, float* out_f, float* out_b, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(flows_f && flows_b && flow_masks && out_f && out_b, "pp_flow_complete_fp32: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_flow_complete<float>(e, flows_f, flows_b, flow_masks, T, H, W, out_f, out_b, 0, 1, as_stream(stream));
}

int pp_flow_complete_dist(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T, int H,
                          int W, float* out_f, float* out_b, int team_first, int team_size, void* stream) {
  return flow_complete_dist<__half>(h, "pp_flow_complete_dist", flows_f, flows_b, flow_masks, T, H, W, out_f, out_b,
                                    team_first, team_size, stream);
}

int pp_flow_complete_dist_fp32(pp_handle h, const float* flows_f, const float* flows_b, const float* flow_masks, int T,
                               int H, int W, float* out_f, float* out_b, int team_first, int team_size, void* stream) {
  return flow_complete_dist<float>(h, "pp_flow_complete_dist_fp32", flows_f, flows_b, flow_masks, T, H, W, out_f,
                                   out_b, team_first, team_size, stream);
}

int pp_image_propagate(pp_handle h, const float* frames, const float* masks, const float* flows_f,
                       const float* flows_b, int T, int H, int W, float* updated_frames, float* updated_masks,
                       void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(frames && masks && flows_f && flows_b && updated_frames && updated_masks,
             "pp_image_propagate: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_image_propagate<__half>(e, frames, masks, flows_f, flows_b, T, H, W, updated_frames, updated_masks,
                                          as_stream(stream));
}

int pp_image_propagate_fp32(pp_handle h, const float* frames, const float* masks, const float* flows_f,
                            const float* flows_b, int T, int H, int W, float* updated_frames, float* updated_masks,
                            void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(frames && masks && flows_f && flows_b && updated_frames && updated_masks,
             "pp_image_propagate_fp32: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_image_propagate<float>(e, frames, masks, flows_f, flows_b, T, H, W, updated_frames, updated_masks,
                                         as_stream(stream));
}

int pp_gen_begin_subset(pp_handle h, const float* updated_frames, const float* masks_dilated,
                        const float* updated_masks, const float* flows_f, const float* flows_b, int T, int H, int W,
                        const unsigned char* frames_needed, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(updated_frames && masks_dilated && updated_masks && flows_f && flows_b, "pp_gen_begin: null pointer");
  const int r = pp_stage_gen_begin(e, updated_frames, masks_dilated, updated_masks, flows_f, flows_b, T, H, W,
                                   frames_needed, as_stream(stream));
  if (r != PP_OK) pp_stage_gen_end(e);   // a failed begin leaves no session and no allocation behind
  return r;
}

int pp_gen_begin(pp_handle h, const float* updated_frames, const float* masks_dilated, const float* updated_masks,
                 const float* flows_f, const float* flows_b, int T, int H, int W, void* stream) {
  return pp_gen_begin_subset(h, updated_frames, masks_dilated, updated_masks, flows_f, flows_b, T, H, W, nullptr, stream);
}

int pp_gen_window(pp_handle h, const int* frame_ids, int t, int l_t, void* pred_f16, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(frame_ids && pred_f16, "pp_gen_window: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_gen_window(e, frame_ids, t, l_t, static_cast<__half*>(pred_f16), as_stream(stream));
}

int pp_gen_run(pp_handle h, const int* frame_ids, const int* win_t, const int* win_lt, int n_windows, void* pred_f16,
               void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(frame_ids && win_t && win_lt && pred_f16, "pp_gen_run: null pointer");
  ArenaGuard guard(e.arena);
  return pp_stage_gen_run(e, frame_ids, win_t, win_lt, n_windows, static_cast<__half*>(pred_f16), as_stream(stream));
}

int pp_gen_end(pp_handle h) {
  PP_HANDLE(h);
  return pp_stage_gen_end(e);
}

int pp_composite(pp_handle h, const void* pred_f16, const float* masks_dilated, const uint8_t* orig, uint8_t* comp,
                 const int* frame_ids_dev, const int* first_visit_dev, int l_t, int H, int W, int half_math,
                 void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(pred_f16 && masks_dilated && orig && comp && frame_ids_dev && first_visit_dev, "pp_composite: null pointer");
  e.launches++;
  return pp_k_composite(static_cast<const __half*>(pred_f16), 4, masks_dilated, orig, comp, frame_ids_dev,
                        first_visit_dev, l_t, H, W, half_math, as_stream(stream));
}

int pp_preprocess(pp_handle h, const float* image, const float* mask, int mask_frames, int T, int H, int W,
                  int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8, float* frames, float* flow_masks,
                  float* masks_dilated, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(image && mask && orig_u8 && frames && flow_masks && masks_dilated, "pp_preprocess: null pointer");
  ArenaGuard guard(e.arena);
  uint8_t* scratch;
  PP_TRY(pp_alloc(e, &scratch, (size_t)mask_frames * H * W, "mask scratch"));
  PP_TRY(pp_k_quantize_frames(image, orig_u8, frames, T, H, W, as_stream(stream)));
  PP_TRY(pp_k_prepare_masks(mask, mask_frames, T, H, W, flow_mask_dilates, mask_dilates, scratch, flow_masks,
                            masks_dilated, as_stream(stream)));
  e.launches += 4;
  return PP_OK;
}

// Coefficient scratch (ints) of pp_k_resize_bicubic_u8 for an H x W -> out_h x out_w resize, both passes
static size_t resize_coef_ints(int H, int W, int out_h, int out_w) {
  const int mx = out_h > out_w ? out_h : out_w;
  const double sc = fmax(fmax((double)H / out_h, (double)W / out_w), 1.0);
  return 2 * (size_t)mx * ((size_t)ceil(2.0 * sc) * 2 + 1 + 2) + 64;
}

// Shared tail of the pre-processing entry points: 8-bit frames / masks at the input size -> outputs at the processing size
static int preprocess_from_u8(PPEngine& e, const uint8_t* u8_in, const uint8_t* m_in, int mask_frames, int T, int H, int W,
                              int out_h, int out_w, int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8, float* frames,
                              float* flow_masks, float* masks_dilated, cudaStream_t st) {
  const bool resize = out_h != H || out_w != W;
  const uint8_t* m_use = m_in;
  if (resize) {
    const size_t mid_px = (size_t)T * H * out_w;
    uint8_t *tmp, *m_out;
    int* coef;
    const size_t coef_ints = resize_coef_ints(H, W, out_h, out_w);
    PP_TRY(pp_alloc(e, &tmp, mid_px * 3, "resize pass 1"));
    PP_TRY(pp_alloc(e, &m_out, (size_t)mask_frames * out_h * out_w, "mask resized"));
    PP_TRY(pp_alloc(e, &coef, coef_ints, "resize coefficients"));
    // frames: bicubic on the 8-bit image (image_utils.py:98-103); masks: the 8-bit 'L' image the same way (:142-150)
    PP_TRY(pp_k_resize_bicubic_u8(u8_in, orig_u8, tmp, coef, coef_ints, T, H, W, 3, out_h, out_w, st));
    PP_TRY(pp_k_resize_bicubic_u8(m_in, m_out, tmp, coef, coef_ints, mask_frames, H, W, 1, out_h, out_w, st));
    m_use = m_out;
    e.launches += 4;
  } else {
    PP_CUDA_CHECK(cudaMemcpyAsync(orig_u8, u8_in, (size_t)T * H * W * 3, cudaMemcpyDeviceToDevice, st));
  }
  PP_TRY(pp_k_u8_to_frames(orig_u8, frames, T, out_h, out_w, st));                       // u8/255*2-1 (:186-190)
  // any non-zero -> dilations (image_utils.py:152-170)
  PP_TRY(pp_k_dilate_masks_u8(m_use, mask_frames, T, out_h, out_w, flow_mask_dilates, mask_dilates, flow_masks,
                              masks_dilated, st));
  e.launches += 3;
  return PP_OK;
}

int pp_preprocess_resize(pp_handle h, const float* image, const float* mask, int mask_frames, int T, int H, int W,
                         int out_h, int out_w, int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8, float* frames,
                         float* flow_masks, float* masks_dilated, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(image && mask && orig_u8 && frames && flow_masks && masks_dilated, "pp_preprocess_resize: null pointer");
  PP_REQUIRE(out_h > 0 && out_w > 0 && H > 0 && W > 0, "pp_preprocess_resize: bad size");
  ArenaGuard guard(e.arena);
  cudaStream_t st = as_stream(stream);
  const size_t in_px = (size_t)T * H * W;
  uint8_t *u8_in, *m_in;
  PP_TRY(pp_alloc(e, &u8_in, in_px * 3, "resize input"));
  PP_TRY(pp_alloc(e, &m_in, (size_t)mask_frames * H * W, "mask input"));
  // float -> uint8 (truncate) for the frames (image_utils.py:106-114) and the mask images (:128-134)
  PP_TRY(pp_k_quantize_u8(image, u8_in, (long long)in_px * 3, st));
  PP_TRY(pp_k_quantize_u8(mask, m_in, (long long)mask_frames * H * W, st));
  e.launches += 2;
  return preprocess_from_u8(e, u8_in, m_in, mask_frames, T, H, W, out_h, out_w, flow_mask_dilates, mask_dilates, orig_u8,
                            frames, flow_masks, masks_dilated, st);
}

int pp_preprocess_u8(pp_handle h, const uint8_t* image_u8, const uint8_t* mask_u8, int mask_frames, int T, int H, int W,
                     int out_h, int out_w, int flow_mask_dilates, int mask_dilates, uint8_t* orig_u8, float* frames,
                     float* flow_masks, float* masks_dilated, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(image_u8 && mask_u8 && orig_u8 && frames && flow_masks && masks_dilated, "pp_preprocess_u8: null pointer");
  PP_REQUIRE(out_h > 0 && out_w > 0 && H > 0 && W > 0, "pp_preprocess_u8: bad size");
  ArenaGuard guard(e.arena);
  return preprocess_from_u8(e, image_u8, mask_u8, mask_frames, T, H, W, out_h, out_w, flow_mask_dilates, mask_dilates,
                            orig_u8, frames, flow_masks, masks_dilated, as_stream(stream));
}

int pp_preprocess_outpaint_u8(pp_handle h, const uint8_t* image_u8, int T, int H, int W, int rw, int rh, int pw, int ph,
                              uint8_t* orig_u8, float* frames, float* flow_masks, float* masks_dilated, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(image_u8 && orig_u8 && frames && flow_masks && masks_dilated, "pp_preprocess_outpaint_u8: null pointer");
  PP_REQUIRE(T > 0 && H > 0 && W > 0 && rw > 0 && rh > 0, "pp_preprocess_outpaint_u8: bad size (T %d, %dx%d -> %dx%d)", T,
             W, H, rw, rh);
  PP_REQUIRE(rw <= pw && rh <= ph, "pp_preprocess_outpaint_u8: the %dx%d frames do not fit the %dx%d canvas", rw, rh, pw,
             ph);
  ArenaGuard guard(e.arena);
  cudaStream_t st = as_stream(stream);
  const uint8_t* window = image_u8;
  if (rw != W || rh != H) {   // PIL's bicubic resize of the 8-bit frames to the processing size (image_utils.py:98-103)
    uint8_t *tmp, *resized;
    int* coef;
    const size_t coef_ints = resize_coef_ints(H, W, rh, rw);
    PP_TRY(pp_alloc(e, &tmp, (size_t)T * H * rw * 3, "resize pass 1"));
    PP_TRY(pp_alloc(e, &resized, (size_t)T * rh * rw * 3, "outpaint window"));
    PP_TRY(pp_alloc(e, &coef, coef_ints, "resize coefficients"));
    PP_TRY(pp_k_resize_bicubic_u8(image_u8, resized, tmp, coef, coef_ints, T, H, W, 3, rh, rw, st));
    window = resized;
    e.launches += (rw != W) + (rh != H);
  }
  PP_TRY(pp_k_outpaint_canvas(window, T, rw, rh, pw, ph, orig_u8, frames, flow_masks, masks_dilated, st));
  e.launches++;
  return PP_OK;
}

// Host helper (no GPU involved): float [0,1] -> uint8 with the reference's arithmetic -- x * 255 in float32, clip to
// [0, 255], truncate (utils/image_utils.py:106-114, 128-134) -- on `threads` host threads.  Lets a host caller ship 1/4 of
// the bytes over PCIe: quantise straight into a page-locked staging buffer, copy, then pp_preprocess_u8.
int pp_host_quantize_u8(const float* src, uint8_t* dst, long long n, int threads) {
  PP_REQUIRE(src != nullptr && dst != nullptr && n >= 0, "pp_host_quantize_u8: bad argument");
  if (threads < 1) threads = 1;
  if (threads > 64) threads = 64;
  auto work = [=](long long lo, long long hi) {
    for (long long i = lo; i < hi; ++i) {
      float v = src[i] * 255.0f;
      v = v < 0.0f ? 0.0f : (v > 255.0f ? 255.0f : v);     // NaN compares false twice and converts to 0 like the device path
      dst[i] = (uint8_t)(int)v;
    }
  };
  if (threads == 1 || n < (1 << 16)) { work(0, n); return PP_OK; }
  std::vector<std::thread> pool;
  const long long per = (n + threads - 1) / threads;
  for (int t = 0; t < threads; ++t) {
    const long long lo = t * per, hi = lo + per < n ? lo + per : n;
    if (lo < hi) pool.emplace_back(work, lo, hi);
  }
  for (auto& th : pool) th.join();
  return PP_OK;
}

int pp_quantize_u8(pp_handle h, const float* src, uint8_t* dst, long long n, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(src && dst && n >= 0, "pp_quantize_u8: bad argument");
  if (n == 0) return PP_OK;
  e.launches++;
  return pp_k_quantize_u8(src, dst, n, as_stream(stream));
}

int pp_postprocess(pp_handle h, const uint8_t* comp_u8, float* image_out, long long n, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(comp_u8 && image_out, "pp_postprocess: null pointer");
  e.launches++;
  return pp_k_u8_to_unit_float(comp_u8, image_out, n, as_stream(stream));
}

long long pp_launch_count(pp_handle h) { return h ? reinterpret_cast<PPEngine*>(h)->launches : 0; }
size_t pp_workspace_peak(pp_handle h) { return h ? reinterpret_cast<PPEngine*>(h)->arena.peak : 0; }

int pp_profile_enable(pp_handle h, int on) {
  PP_HANDLE(h);
  PP_CUDA_CHECK(cudaDeviceSynchronize());
  for (auto& r : e.prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  e.prof.clear();
  e.profile = on != 0;
  return PP_OK;
}

// Writes "name\tcount\tms\trows\tflops\tbytes\n" per kernel name (aggregated) into buf.
int pp_profile_dump(pp_handle h, char* buf, size_t cap) {
  PP_HANDLE(h);
  PP_REQUIRE(buf != nullptr && cap > 0, "pp_profile_dump: no buffer");
  PP_CUDA_CHECK(cudaDeviceSynchronize());
  struct Agg { long long n = 0; double ms = 0, rows = 0, flops = 0, bytes = 0; };
  std::map<std::string, Agg> agg;
  for (auto& r : e.prof) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) ms = 0.f;
    Agg& a = agg[r.name];
    a.n++; a.ms += ms; a.rows += r.rows; a.flops += r.flops; a.bytes += r.bytes;
  }
  size_t off = 0;
  buf[0] = 0;
  for (auto& kv : agg) {
    char line[512];
    int n = snprintf(line, sizeof(line), "%s\t%lld\t%.6f\t%.0f\t%.0f\t%.0f\n", kv.first.c_str(), kv.second.n,
                     kv.second.ms, kv.second.rows, kv.second.flops, kv.second.bytes);
    if (off + n + 1 > cap) { pp_set_error("pp_profile_dump: buffer too small"); return PP_ERR_ARG; }
    memcpy(buf + off, line, n + 1);
    off += n;
  }
  return PP_OK;
}

// ---- single-operator entry points --------------------------------------------------------------------
int pp_op_conv(pp_handle h, const char* name, const void* x_f16, int N, int H, int W, int stride, int pad, int dil,
               int replicate, int act, float slope, const void* residual_f16, void* out_f16, void* stream) {
  PP_HANDLE(h);
  const PPPackedConv* w = nullptr;
  PP_TRY(pp_get_conv(e, name, &w));
  PPConvCall c(e, name, N, H, W);
  c.in(static_cast<const __half*>(x_f16), w->cin_g * w->groups, 0, w->cin_g, w->groups > 1 ? w->cin_g : 0)
      .geom(stride, stride, pad, pad, dil, dil, replicate)
      .out(static_cast<__half*>(out_f16), w->cout_g * w->groups, 0, w->groups > 1 ? w->cout_g : 0)
      .act(act, slope);
  if (residual_f16 != nullptr) c.residual(static_cast<const __half*>(residual_f16), w->cout_g * w->groups, 0);
  return c.run(as_stream(stream));
}

int pp_op_conv_ex(pp_handle h, const char* name, const void* x_f16, int x_C, int x_co, int N, int H, int W, int ph,
                  int pw, int epi, int act, float slope, float scale, int act2, const void* aux0_f16, int aux0_C,
                  int aux0_co, void* aux1_f16, int aux1_C, int aux1_co, void* out_f16, int out_C, int out_co, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(name && x_f16 && out_f16, "pp_op_conv_ex: null pointer");
  PP_REQUIRE(epi == PP_EPI_STD || (aux0_f16 && aux1_f16), "pp_op_conv_ex: the GRU epilogues need aux0 and aux1");
  const PPPackedConv* w = nullptr;
  PP_TRY(pp_get_conv(e, name, &w));
  PPConvCall c(e, name, N, H, W);
  c.in(static_cast<const __half*>(x_f16), x_C, x_co, w->cin_g, w->groups > 1 ? w->cin_g : 0)
      .geom(1, 1, ph, pw)
      .out(static_cast<__half*>(out_f16), out_C, out_co, w->groups > 1 ? w->cout_g : 0);
  const __half* a0 = static_cast<const __half*>(aux0_f16);
  __half* a1 = static_cast<__half*>(aux1_f16);
  if (epi == PP_EPI_GRU_ZR) {
    c.gru_zr(a0, aux0_C, aux0_co, a1, aux1_C, aux1_co);
  } else if (epi == PP_EPI_GRU_H) {
    c.gru_h(a0, aux0_C, aux0_co, a1, aux1_C, aux1_co);
  } else {
    c.act(act, slope, scale, act2);
    if (a0 != nullptr) c.residual(a0, aux0_C, aux0_co);
  }
  return c.run(as_stream(stream));
}

int pp_op_conv_segs(pp_handle h, const char* name, int nseg, const void* const* x_f16, const int* x_C, const int* x_co,
                    const int* x_ch, const int* x_gstep, int N, int H, int W, int sh, int sw, int ph, int pw, int dh,
                    int dw, int replicate, int epi, int act, float slope, float scale, int act2, const void* aux0_f16,
                    int aux0_C, int aux0_co, void* aux1_f16, int aux1_C, int aux1_co, void* out, int out_C, int out_co,
                    int out_gstep, int out_fp32, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(name && x_f16 && x_C && x_co && x_ch && x_gstep && out, "pp_op_conv_segs: null pointer");
  PP_REQUIRE(nseg >= 1 && nseg <= PP_MAX_SEGS, "pp_op_conv_segs: %d input segments (1..%d)", nseg, PP_MAX_SEGS);
  PP_REQUIRE(epi == PP_EPI_STD || (aux0_f16 && aux1_f16 && !out_fp32),
             "pp_op_conv_segs: the GRU epilogues need aux0 and aux1 and an fp16 output");
  PPConvCall c(e, name, N, H, W);
  for (int i = 0; i < nseg; ++i) c.in(static_cast<const __half*>(x_f16[i]), x_C[i], x_co[i], x_ch[i], x_gstep[i]);
  c.geom(sh, sw, ph, pw, dh, dw, replicate);
  if (out_fp32) c.out_f32(static_cast<float*>(out), out_C, out_co);
  else c.out(static_cast<__half*>(out), out_C, out_co, out_gstep);
  const __half* a0 = static_cast<const __half*>(aux0_f16);
  __half* a1 = static_cast<__half*>(aux1_f16);
  if (epi == PP_EPI_GRU_ZR) {
    c.gru_zr(a0, aux0_C, aux0_co, a1, aux1_C, aux1_co);
  } else if (epi == PP_EPI_GRU_H) {
    c.gru_h(a0, aux0_C, aux0_co, a1, aux1_C, aux1_co);
  } else {
    c.act(act, slope, scale, act2);
    if (a0 != nullptr) c.residual(a0, aux0_C, aux0_co);
  }
  return c.run(as_stream(stream));
}

int pp_op_conv_last_plan(int* plan, int n) {
  PP_REQUIRE(plan != nullptr && n >= 0, "pp_op_conv_last_plan: bad argument");
  const PPConvPlan& p = pp_last_conv_plan();
  const int v[8] = {p.kind, p.m, p.bn, p.tps, p.flat, p.tma_out, p.sa, p.sb};
  for (int i = 0; i < n && i < 8; ++i) plan[i] = v[i];
  return PP_OK;
}

int pp_op_corr_lookup(pp_handle h, const void* l0, const void* l1, const void* l2, const void* l3,
                      const float* coords, void* out_f16, long long nq, int h8, int w8, void* stream) {
  PP_HANDLE(h);
  e.launches++;
  return pp_k_corr_lookup(static_cast<const __half*>(l0), static_cast<const __half*>(l1),
                          static_cast<const __half*>(l2), static_cast<const __half*>(l3), coords,
                          static_cast<__half*>(out_f16), 328, nq, h8, w8, as_stream(stream));
}

int pp_op_conv_tf32(pp_handle h, const char* name, const float* x0, int x0_C, int x0_co, int x0_ch, const float* x1,
                    int x1_C, int x1_co, int x1_ch, int N, int H, int W, int sh, int sw, int ph, int pw, int dh, int dw,
                    int replicate, int epi, int act, float slope, float scale, int act2, const float* aux0, int aux0_C, int aux0_co, float* aux1,
                    int aux1_C, int aux1_co, float* out, int out_C, int out_co, int out_fp32, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(name && x0 && out, "pp_op_conv_tf32: null pointer");
  PP_REQUIRE(epi == PP_EPI_STD || (aux0 && aux1), "pp_op_conv_tf32: the GRU epilogues need aux0 and aux1");
  PPConvCall c(e, name, N, H, W);
  c.in(x0, x0_C, x0_co, x0_ch);
  if (x1 != nullptr) c.in(x1, x1_C, x1_co, x1_ch);
  c.geom(sh, sw, ph, pw, dh, dw, replicate);
  if (out_fp32) c.out_f32(out, out_C, out_co);
  else c.out(out, out_C, out_co);
  if (epi == PP_EPI_GRU_ZR) {
    c.gru_zr(aux0, aux0_C, aux0_co, aux1, aux1_C, aux1_co);
  } else if (epi == PP_EPI_GRU_H) {
    c.gru_h(aux0, aux0_C, aux0_co, aux1, aux1_C, aux1_co);
  } else {
    c.act(act, slope, scale, act2);
    if (aux0 != nullptr) c.residual(aux0, aux0_C, aux0_co);
  }
  return c.run(as_stream(stream));
}

int pp_op_dcn_sample_f32(pp_handle h, const float* x0, int C0, const float* x1, int C1, const float* offs, int N,
                         int H, int W, float max_mag, float* cols, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(al16(x0) && al16(x1) && al16(cols), "pp_op_dcn_sample_f32: x0, x1 and cols must be 16-byte aligned");
  e.launches++;
  return pp_k_dcn_sample(x0, C0, x1, C1, offs, 432, max_mag, cols, N, H, W, as_stream(stream));
}

int pp_op_upsample2x_f32(pp_handle h, const float* src, float* dst, int N, int H, int W, int C, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(src && dst, "pp_op_upsample2x_f32: null pointer");
  PP_REQUIRE(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0,
             "pp_op_upsample2x_f32: src and dst must be 16-byte aligned");
  e.launches++;
  return pp_k_upsample2x(src, dst, N, H, W, C, as_stream(stream));
}

int pp_op_instnorm(pp_handle h, const void* x, const void* residual, void* out, int N, int HW, int C, int relu, int fp32,
                   void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(x && out, "pp_op_instnorm: null pointer");
  return fp32 ? op_instnorm<float>(e, x, residual, out, N, HW, C, relu, as_stream(stream))
              : op_instnorm<__half>(e, x, residual, out, N, HW, C, relu, as_stream(stream));
}

int pp_op_corr_pyramid(pp_handle h, const void* fmap1, const void* fmap2, int pairs, int h8, int w8, int fp32, void* l0,
                       void* l1, void* l2, void* l3, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(fmap1 && fmap2 && l0 && l1 && l2 && l3 && pairs >= 1, "pp_op_corr_pyramid: bad argument");
  return fp32 ? op_corr_pyramid<float>(e, fmap1, fmap2, pairs, h8, w8, l0, l1, l2, l3, as_stream(stream))
              : op_corr_pyramid<__half>(e, fmap1, fmap2, pairs, h8, w8, l0, l1, l2, l3, as_stream(stream));
}

int pp_op_corr_lookup_f32(pp_handle h, const float* l0, const float* l1, const float* l2, const float* l3,
                          const float* coords, float* out, long long nq, int h8, int w8, void* stream) {
  PP_HANDLE(h);
  e.launches++;
  return pp_k_corr_lookup(l0, l1, l2, l3, coords, out, 352, nq, h8, w8, as_stream(stream));
}

int pp_op_convex_upsample(pp_handle h, const float* coords1, const void* mask, float* out, int B, int h8, int w8, int fp32,
                          void* stream) {
  PP_HANDLE(h);
  e.launches++;
  if (fp32) return pp_k_convex_upsample(coords1, static_cast<const float*>(mask), out, B, h8, w8, as_stream(stream));
  return pp_k_convex_upsample(coords1, static_cast<const __half*>(mask), out, B, h8, w8, as_stream(stream));
}

int pp_op_imgprop_step(pp_handle h, const void* cur4_f16, const void* prop_in4_f16, void* prop_out4_f16,
                       const void* flow_prop_f16, const void* flow_check_f16, int H, int W, void* stream) {
  PP_HANDLE(h);
  e.launches++;
  return pp_k_imgprop_step(static_cast<const __half*>(cur4_f16), static_cast<const __half*>(prop_in4_f16),
                           static_cast<__half*>(prop_out4_f16), static_cast<const __half*>(flow_prop_f16),
                           static_cast<const __half*>(flow_check_f16), H, W, as_stream(stream));
}

int pp_op_imgprop_step_f32(pp_handle h, const float* cur4, const float* prop_in4, float* prop_out4,
                           const float* flow_prop, const float* flow_check, int H, int W, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(cur4 && prop_in4 && prop_out4 && flow_prop && flow_check, "pp_op_imgprop_step_f32: null pointer");
  e.launches++;
  return pp_k_imgprop_step(cur4, prop_in4, prop_out4, flow_prop, flow_check, H, W, as_stream(stream));
}

int pp_op_attention(pp_handle h, const void* qkv_f16, const void* pkv_f16, void* out_f16, const int* win_flags_dev,
                    const int* win_t, int n_windows, int gh, int gw, int n_pool, int parity, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(qkv_f16 && pkv_f16 && out_f16 && win_flags_dev && win_t && n_windows >= 1, "pp_op_attention: bad argument");
  PP_REQUIRE(al16(qkv_f16) && al16(pkv_f16) && al16(out_f16), "pp_op_attention: qkv, pkv and out must be 16-byte aligned");
  const int nh = pp_ceil_div(gh, 5) * 5, nw = pp_ceil_div(gw, 9) * 9;
  // the sliding windows' frames are concatenated: window w owns frames [foff[w], foff[w] + t[w]) (pp_stage_gen_run)
  std::vector<int> meta(2 * n_windows);
  int t_max = 0;
  for (int w = 0, off = 0; w < n_windows; ++w) {
    PP_REQUIRE(win_t[w] >= 2, "pp_op_attention: window %d has t=%d (< 2)", w, win_t[w]);
    meta[w] = off;
    meta[n_windows + w] = win_t[w];
    off += win_t[w];
    if (win_t[w] > t_max) t_max = win_t[w];
  }
  std::vector<int> ring;
  pp_build_ring_indices(nh, nw, ring);
  ArenaGuard guard(e.arena);
  cudaStream_t st = as_stream(stream);
  int *ring_dev, *meta_dev, *key_tab;
  PP_TRY(pp_alloc(e, &ring_dev, ring.size(), "ring indices"));
  PP_CUDA_CHECK(cudaMemcpyAsync(ring_dev, ring.data(), ring.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  PP_TRY(pp_alloc(e, &meta_dev, meta.size(), "attention meta"));
  PP_CUDA_CHECK(cudaMemcpyAsync(meta_dev, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const int key_stride = ((t_max + 1) / 2) * (193 + n_pool);
  PP_TRY(pp_alloc(e, &key_tab, (size_t)(nh / 5) * (nw / 9) * key_stride, "attention key table"));
  const __half* qkv = static_cast<const __half*>(qkv_f16);
  const __half* pkv = static_cast<const __half*>(pkv_f16);
  PP_TRY(pp_k_attention(qkv, qkv + 512, qkv + 1024, 1536, pkv, pkv + 512, 1024, static_cast<__half*>(out_f16), 512,
                        win_flags_dev, ring_dev, meta_dev, meta_dev + n_windows, n_windows, t_max, gh, gw, nh, nw, n_pool,
                        parity, key_tab, key_stride, st));
  e.launches++;
  PP_CUDA_CHECK(cudaStreamSynchronize(st));   // the scratch goes back to the arena on return
  return PP_OK;
}

int pp_op_layernorm(pp_handle h, const void* x_f16, const float* gamma, const float* beta, void* out_f16, int t, int gh,
                    int gw, int nh, int nw, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(x_f16 && gamma && beta && out_f16, "pp_op_layernorm: null pointer");
  PP_REQUIRE(al16(x_f16) && al16(gamma) && al16(beta) && al16(out_f16),
             "pp_op_layernorm: x, gamma, beta and out must be 16-byte aligned");
  PP_REQUIRE(t >= 0 && gh >= 1 && gw >= 1 && nh >= gh && nw >= gw, "pp_op_layernorm: grid %dx%d in %dx%d", gh, gw, nh, nw);
  e.launches++;
  return pp_k_layernorm(static_cast<const __half*>(x_f16), gamma, beta, static_cast<__half*>(out_f16),
                        (long long)t * gh * gw, gh, gw, nh, nw, as_stream(stream));
}

int pp_op_pool_tokens(pp_handle h, const void* x_f16, const float* w, const float* b, void* out_f16, int t, int nh,
                      int nw, int C, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(x_f16 && w && b && out_f16, "pp_op_pool_tokens: null pointer");
  PP_REQUIRE(al16(x_f16) && al16(w) && al16(b) && al16(out_f16), "pp_op_pool_tokens: x, w, b and out must be 16-byte aligned");
  PP_REQUIRE(nh >= 4 && nw >= 4, "pp_op_pool_tokens: grid %dx%d is smaller than the 4x4 pooling window", nh, nw);
  e.launches++;
  return pp_k_pool_tokens(static_cast<const __half*>(x_f16), w, b, static_cast<__half*>(out_f16), t, nh, nw,
                          (nh - 4) / 4 + 1, (nw - 4) / 4 + 1, C, as_stream(stream));
}

int pp_op_window_flags(pp_handle h, const void* mask4_f16, int cs, int co, const int* win_f0, const int* win_lt,
                       int n_windows, int h4, int w4, int* flags_dev, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(mask4_f16 && win_f0 && win_lt && flags_dev && n_windows >= 1 && h4 >= 1 && w4 >= 1 && co < cs,
             "pp_op_window_flags: bad argument");
  const int gh = (h4 - 1) / 3 + 1, gw = (w4 - 1) / 3 + 1;   // unfold(7, stride 3, pad 3) token grid
  std::vector<int> meta(win_f0, win_f0 + n_windows);
  meta.insert(meta.end(), win_lt, win_lt + n_windows);
  ArenaGuard guard(e.arena);
  cudaStream_t st = as_stream(stream);
  int* meta_dev;
  PP_TRY(pp_alloc(e, &meta_dev, meta.size(), "window flag meta"));
  PP_CUDA_CHECK(cudaMemcpyAsync(meta_dev, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  PP_TRY(pp_k_window_flags(static_cast<const __half*>(mask4_f16), cs, co, meta_dev, meta_dev + n_windows, n_windows, h4,
                           w4, gh, gw, pp_ceil_div(gh, 5), pp_ceil_div(gw, 9), flags_dev, st));
  e.launches++;
  PP_CUDA_CHECK(cudaStreamSynchronize(st));
  return PP_OK;
}

int pp_op_fold(pp_handle h, const void* x_f16, int cs, void* out_f16, int t, int H, int W, int C, int normalise, int gelu,
               void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(x_f16 && out_f16 && H >= 1 && W >= 1 && C <= cs / 49, "pp_op_fold: bad argument (C=%d cs=%d)", C, cs);
  PP_REQUIRE(al16(x_f16) && al16(out_f16), "pp_op_fold: x and out must be 16-byte aligned");
  e.launches++;
  return pp_k_fold(static_cast<const __half*>(x_f16), cs, static_cast<__half*>(out_f16), t, H, W, C, (H - 1) / 3 + 1,
                   (W - 1) / 3 + 1, normalise, gelu, as_stream(stream));
}

int pp_op_featprop_cond(pp_handle h, const void* cur_f16, const void* prop_f16, const void* flow_prop_f16,
                        const void* flow_check_f16, const void* mask2_f16, void* cond_f16, int N, int H, int W,
                        void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(cur_f16 && prop_f16 && flow_prop_f16 && flow_check_f16 && mask2_f16 && cond_f16,
             "pp_op_featprop_cond: null pointer");
  PP_REQUIRE(al16(cur_f16) && al16(prop_f16) && al16(mask2_f16) && al16(cond_f16) &&
                 ((reinterpret_cast<uintptr_t>(flow_prop_f16) | reinterpret_cast<uintptr_t>(flow_check_f16)) & 3) == 0,
             "pp_op_featprop_cond: cur, prop, mask2 and cond must be 16-byte aligned, the flows 4-byte aligned");
  e.launches++;
  return pp_k_featprop_cond(static_cast<const __half*>(cur_f16), 128, static_cast<const __half*>(prop_f16), 128,
                            static_cast<const __half*>(flow_prop_f16), static_cast<const __half*>(flow_check_f16),
                            static_cast<const __half*>(mask2_f16), 8, static_cast<__half*>(cond_f16), 264, N, H, W, 128,
                            as_stream(stream));
}

int pp_op_dcn_sample(pp_handle h, const void* x0_f16, int x0_cs, int C0, const void* x1_f16, int x1_cs, int C1,
                     const void* offs_f16, const void* flow_f16, int flow_cs, int flow_co, float max_mag, void* cols_f16,
                     int N, int H, int W, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(x0_f16 && offs_f16 && cols_f16 && (C1 == 0 || x1_f16), "pp_op_dcn_sample: null pointer");
  PP_REQUIRE(al16(x0_f16) && al16(x1_f16) && al16(cols_f16) && x0_cs % 8 == 0 && (C1 == 0 || x1_cs % 8 == 0),
             "pp_op_dcn_sample: x0, x1 and cols must be 16-byte aligned with channel strides that are multiples of 8");
  PP_REQUIRE(C0 <= x0_cs && (C1 == 0 || C1 <= x1_cs), "pp_op_dcn_sample: channels exceed the channel strides");
  PP_REQUIRE(flow_f16 == nullptr || flow_co + 2 <= flow_cs, "pp_op_dcn_sample: flow channels %d..%d of %d", flow_co,
             flow_co + 1, flow_cs);
  e.launches++;
  return pp_k_dcn_sample(static_cast<const __half*>(x0_f16), x0_cs, 0, C0, static_cast<const __half*>(x1_f16), x1_cs, 0,
                         C1, static_cast<const __half*>(offs_f16), 432, static_cast<const __half*>(flow_f16), flow_cs,
                         flow_co, max_mag, static_cast<__half*>(cols_f16), N, H, W, as_stream(stream));
}

int pp_op_downsample4(pp_handle h, const float* flows, void* flows4_f16, int n_flows, const float* masks,
                      void* masks4_f16, int mask_co, int n_masks, int H, int W, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE((flows == nullptr) == (flows4_f16 == nullptr) && (masks == nullptr) == (masks4_f16 == nullptr) &&
                 mask_co >= 0 && mask_co < 8,
             "pp_op_downsample4: bad argument");
  PP_REQUIRE(H % 4 == 0 && W % 4 == 0, "pp_op_downsample4: size %dx%d must be a multiple of 4", W, H);
  PP_REQUIRE((reinterpret_cast<uintptr_t>(flows4_f16) & 3) == 0, "pp_op_downsample4: flows4 must be 4-byte aligned");
  cudaStream_t st = as_stream(stream);
  if (flows != nullptr) {
    PP_TRY(pp_k_downsample_flow4(flows, static_cast<__half*>(flows4_f16), n_flows, H, W, st));
    e.launches++;
  }
  if (masks != nullptr) {
    PP_TRY(pp_k_downsample_mask4(masks, static_cast<__half*>(masks4_f16), 8, mask_co, n_masks, H, W, st));
    e.launches++;
  }
  return PP_OK;
}

int pp_op_upsample2x(pp_handle h, const void* src_f16, void* dst_f16, int N, int H, int W, int C, void* stream) {
  PP_HANDLE(h);
  PP_REQUIRE(src_f16 && dst_f16, "pp_op_upsample2x: null pointer");
  PP_REQUIRE(al16(src_f16) && al16(dst_f16), "pp_op_upsample2x: src and dst must be 16-byte aligned");
  e.launches++;
  return pp_k_upsample2x(static_cast<const __half*>(src_f16), C, 0, static_cast<__half*>(dst_f16), C, 0, N, H, W, C,
                         as_stream(stream));
}

}  // extern "C"

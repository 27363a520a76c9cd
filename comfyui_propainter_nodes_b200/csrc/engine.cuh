// Engine handle: packed weights registry, workspace arena, conv-call builder, stage entry points.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "conv_igemm.cuh"
#include "kernels.cuh"

struct PPPackedConv {
  const __half* w = nullptr;   // swizzled tile image [groups][num_kc][cout_g_pad][64]
  const float* b = nullptr;    // [groups*cout_g] or null
  int cout_g = 0, cout_g_pad = 0, bn = 0, cin_g = 0, kh = 1, kw = 1, groups = 1;
  // multiply-adds per output pixel of the REFERENCE layer (unpadded channels, real group structure); 0 = unknown,
  // the bench then falls back to the packed shape.  Only used for the roofline's algorithmic flop count.
  double macs_per_pixel = 0.0;
};

struct PPTensor {
  const void* ptr = nullptr;
  size_t bytes = 0;
};

// Bump allocator over one device allocation; stage code uses mark()/release() in stack order.
struct PPArena {
  uint8_t* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  void* alloc(size_t bytes) {
    const size_t a = (off + 255) & ~size_t(255);
    if (a + bytes > cap) return nullptr;
    off = a + bytes;
    if (off > peak) peak = off;
    return base + a;
  }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
};

struct PPEngine {
  int device = 0;
  std::map<std::string, PPPackedConv> convs;
  std::map<std::string, PPTensor> tensors;
  PPArena arena;
  // generator session state (encoder features cached per frame, see generator.cu)
  struct GenSession {
    bool active = false;
    int T = 0, H = 0, W = 0;
    __half* enc = nullptr;        // [T][H/4][W/4][128]
    __half* flows_f4 = nullptr;   // [T-1][h][w][2] (dx,dy)/4
    __half* flows_b4 = nullptr;
    __half* mask_in4 = nullptr;   // [T][h][w] fp16
    size_t arena_mark = 0;
    std::vector<int> ring_idx_host;
    int* ring_idx = nullptr;      // [n_win][193]
    int gh = 0, gw = 0, nh = 0, nw = 0, ph = 0, pw = 0;
  } gen;
  // multi-GPU (comm.cu): NCCL communicator (ncclComm_t, opaque here) of this engine's process group
  void* comm = nullptr;
  int rank = 0, world = 1;
  // multi-layer programs (conv_halo.cu): barrier counter word on the device + arrivals issued on it so far
  unsigned int* prog_counter = nullptr;
  unsigned int prog_arrivals = 0;
  double prog_flops = 0.0;   // algorithmic flops of the layers recorded since pp_prog_begin (profiling)
  long long launches = 0;  // kernels launched by this engine (for bench accounting)
  // optional per-kernel timing (CUDA events on the launch stream), see pp_profile_* in capi.cu
  struct ProfRec {
    std::string name;
    cudaEvent_t a, b;
    double rows, flops, bytes;
  };
  bool profile = false;
  std::vector<ProfRec> prof;
};

// Times one kernel launch when profiling is enabled (events recorded on the launch stream).
struct PPProfScope {
  PPEngine& e;
  cudaStream_t st;
  bool on;
  PPProfScope(PPEngine& eng, const std::string& name, double rows, double flops, double bytes, cudaStream_t s)
      : e(eng), st(s), on(eng.profile) {
    if (!on) return;
    PPEngine::ProfRec r;
    r.name = name; r.rows = rows; r.flops = flops; r.bytes = bytes;
    cudaEventCreate(&r.a);
    cudaEventCreate(&r.b);
    cudaEventRecord(r.a, st);
    e.prof.push_back(r);
  }
  ~PPProfScope() {
    if (on) cudaEventRecord(e.prof.back().b, st);
  }
};

template <typename T>
inline int pp_alloc(PPEngine& e, T** out, size_t count, const char* what) {
  *out = reinterpret_cast<T*>(e.arena.alloc(count * sizeof(T)));
  if (*out == nullptr) {
    pp_set_error("workspace exhausted allocating %s (%zu bytes, used %zu of %zu); raise workspace_bytes in pp_create",
                 what, count * sizeof(T), e.arena.off, e.arena.cap);
    return PP_ERR_STATE;
  }
  return PP_OK;
}

int pp_get_conv(PPEngine& e, const std::string& name, const PPPackedConv** out);
int pp_get_tensor(PPEngine& e, const std::string& name, const void** out);

// Fluent builder around PPConvParams.
struct PPConvCall {
  PPConvParams p;
  PPEngine* eng;
  std::string name;
  int err = PP_OK;
  PPConvCall(PPEngine& e, const std::string& name, int N, int H, int W);
  PPConvCall& in(const __half* ptr, int cs, int co, int channels, int gstep = 0);
  PPConvCall& geom(int sh, int sw, int ph, int pw, int dh = 1, int dw = 1, int replicate = 0);
  PPConvCall& out(__half* ptr, int cs, int co, int gstep = 0);
  PPConvCall& out_f32(float* ptr, int cs, int co);   // plain fp32 [pix][cs] output of either form
  PPConvCall& act(int act1, float slope = 0.f, float scale = 1.f, int act2 = PP_ACT_NONE);
  PPConvCall& residual(const __half* ptr, int cs, int co);
  PPConvCall& gru_zr(const __half* h, int h_cs, int h_co, __half* rh, int rh_cs, int rh_co);
  PPConvCall& gru_h(const __half* h, int h_cs, int h_co, const __half* z, int z_cs, int z_co);
  // Split-tf32 form (PPConvParams::split, conv_igemm.cuh): the float* overloads.  A float* input puts the call in this
  // form; the weights must have been registered as a split image and every input must then be a float* one.  Every
  // tensor is an fp32 [pix][hi C | lo C] pair tensor given by its pointer and real channel count C; `co` / `channels`
  // count fp32 channels.  The inputs are read as (hi..., lo..., hi...) segments by run().
  PPConvCall& in(const float* ptr, int C, int co, int channels);
  PPConvCall& out(float* ptr, int C, int co);
  PPConvCall& residual(const float* ptr, int C, int co);
  PPConvCall& gru_zr(const float* h, int h_C, int h_co, float* rh, int rh_C, int rh_co);
  PPConvCall& gru_h(const float* h, int h_C, int h_co, const float* z, int z_C, int z_co);
  int run(cudaStream_t st);

 private:
  struct SplitIn { const float* ptr; int C, co, channels; };
  SplitIn split_in[PP_MAX_SEGS / 3];
  int n_split_in = 0;
};

void pp_build_ring_indices(int nh, int nw, std::vector<int>& out);

// ---- multi-GPU exchange (comm.cu) -----------------------------------------------------------------
int pp_comm_unique_id_impl(void* out128);
int pp_comm_init_impl(PPEngine& e, const void* unique_id, int rank, int world);
int pp_comm_destroy_impl(PPEngine& e);
int pp_comm_all_gather_blocks_impl(PPEngine& e, void* buf, const long long* row_offset, const long long* rows,
                                   size_t row_bytes, int first_rank, int n_members, cudaStream_t st);

// ---- stages ---------------------------------------------------------------------------------------
// The stages that exist in two precisions are templates on the element type E of their activations, instantiated for
// __half (fp16) and float (the node's fp16="disable"); the C entry points (capi.cu) choose it.
// RAFT, E = float: the split-tf32 path, weights registered under "<name>.tf32" (engine.py).
template <class E>
int pp_stage_raft(PPEngine& e, const float* frames, int T, int H, int W, int iters, float* flows_f, float* flows_b,
                  cudaStream_t st);
// RAFT correlation pyramid (raft.cu), shared by pp_stage_raft and pp_op_corr_pyramid.  P_pad: rows of a packed fmap
// (pp_k_pack_b_operand) of P pixels.
int pp_raft_corr_pad(int P);
// All-pairs correlation of `pairs` frame pairs, scaled by 1/sqrt(256): group g correlates fmap g after fmap1 (fp16
// [P][256], or fp32 split [P][hi 256 | lo 256]) with packed fmap g after fpack2 into corr0 + g*P*P (fp16 / fp32).
template <class E>
int pp_raft_corr_volume(PPEngine& e, const E* fmap1, const E* fpack2, int pairs, int P, int P_pad, E* corr0,
                        cudaStream_t st);
// Levels 1..3 from level 0: 2x2 average pooling of each of the M query maps of h8 x w8
template <class E>
int pp_raft_corr_pool(PPEngine& e, E* const corr[4], long long M, int h8, int w8, cudaStream_t st);
// Flow completion, E = float: split-tf32 activations, weights registered under "<name>.tf32" (engine.py)
template <class E>
int pp_stage_flow_complete(PPEngine& e, const float* flows_f, const float* flows_b, const float* flow_masks, int T,
                           int H, int W, float* out_f, float* out_b, int team_first, int team_size, cudaStream_t st);
// E = float: frames / masks stored as float4 and flows as float2, E = __half: 4 x fp16 / __half2
template <class E>
int pp_stage_image_propagate(PPEngine& e, const float* frames, const float* masks, const float* flows_f,
                             const float* flows_b, int T, int H, int W, float* upd_frames, float* upd_masks,
                             cudaStream_t st);
int pp_stage_gen_begin(PPEngine& e, const float* frames, const float* masks_in, const float* masks_upd,
                 const float* flows_f, const float* flows_b, int T, int H, int W, const unsigned char* need,
                 cudaStream_t st);
int pp_stage_gen_window(PPEngine& e, const int* frame_ids, int t, int l_t, __half* pred /*[l_t][H][W][4]*/,
                  cudaStream_t st);
int pp_stage_gen_run(PPEngine& e, const int* frame_ids, const int* win_t, const int* win_lt, int n_windows,
                     __half* pred /*[sum l_t][H][W][4]*/, cudaStream_t st);
int pp_stage_gen_end(PPEngine& e);

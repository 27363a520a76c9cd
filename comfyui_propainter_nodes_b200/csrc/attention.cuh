// Shared parameter block of the two window-attention kernels (attention.cu: mma.sync, unmasked windows;
// attention_tc.cu: wgmma, masked windows).
#pragma once
#include "pp_common.cuh"

struct PPAttnParams {
  const __half* q; const __half* k; const __half* v; int qkv_cs;  // padded token grid [t][nh*nw][cs]
  const __half* pk; const __half* pv; int pool_cs;                // pooled tokens [t][n_pool][cs]
  __half* out; int out_cs;                                        // unpadded grid [t][gh*gw][cs]
  const int* win_flags;                                           // [n_sliding][n_win] 1 = masked window
  const int* ring_idx;                                            // [n_win][193] token index in padded grid
  const int* sw_frame_off;                                        // [n_sliding] first frame of each sliding window
  const int* sw_t;                                                // [n_sliding] frames in each sliding window
  int n_win, gh, gw, nh, nw, nww, n_pool, parity;
  int only_unmasked;                                              // mma.sync kernel: skip masked windows
  const int* key_tab; int key_tab_stride;                         // [n_win][stride] gather table scratch (attention_tc.cu)
  float scale_log2;
};

int pp_launch_attention_tc(const PPAttnParams& p, int n_sliding, int t_max, cudaStream_t st);

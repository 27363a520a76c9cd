// Engine plumbing: registries and the conv-call builder.
#include <stdlib.h>
#include <string.h>

#include "engine.cuh"

int pp_get_conv(PPEngine& e, const std::string& name, const PPPackedConv** out) {
  auto it = e.convs.find(name);
  if (it == e.convs.end()) {
    pp_set_error("conv weights '%s' were not registered (pp_register_conv)", name.c_str());
    return PP_ERR_STATE;
  }
  *out = &it->second;
  return PP_OK;
}

int pp_get_tensor(PPEngine& e, const std::string& name, const void** out) {
  auto it = e.tensors.find(name);
  if (it == e.tensors.end()) {
    pp_set_error("tensor '%s' was not registered (pp_register_tensor)", name.c_str());
    return PP_ERR_STATE;
  }
  *out = it->second.ptr;
  return PP_OK;
}

PPConvCall::PPConvCall(PPEngine& e, const std::string& name_, int N, int H, int W) : eng(&e), name(name_) {
  memset(&p, 0, sizeof(p));
  const PPPackedConv* w = nullptr;
  err = pp_get_conv(e, name, &w);
  if (err != PP_OK) return;
  p.N = N; p.H = H; p.W = W;
  p.kh = w->kh; p.kw = w->kw;
  p.sh = p.sw = 1; p.dh = p.dw = 1;
  p.ph = (w->kh - 1) / 2; p.pw = (w->kw - 1) / 2;
  p.Cin = w->cin_g;
  p.wpacked = w->w; p.bias = w->b;
  p.Cout_g = w->cout_g; p.Cout_g_pad = w->cout_g_pad; p.BN = w->bn; p.groups = w->groups;
  p.epi = PP_EPI_STD; p.act1 = PP_ACT_NONE; p.act2 = PP_ACT_NONE; p.slope = 0.f; p.scale = 1.f;
  p.nseg = 0;
}

PPConvCall& PPConvCall::in(const __half* ptr, int cs, int co, int channels, int gstep) {
  if (err != PP_OK) return *this;
  if (p.nseg >= PP_MAX_SEGS) { pp_set_error("conv: more than %d input segments", PP_MAX_SEGS); err = PP_ERR_ARG; return *this; }
  PPConvSeg& s = p.seg[p.nseg];
  s.ptr = ptr; s.cstride = cs; s.coff = co; s.gstep = gstep;
  s.cbegin = p.nseg == 0 ? 0 : p.seg[p.nseg - 1].cend;
  s.cend = s.cbegin + channels;
  ++p.nseg;
  return *this;
}

PPConvCall& PPConvCall::geom(int sh, int sw, int ph, int pw, int dh, int dw, int replicate) {
  p.sh = sh; p.sw = sw; p.ph = ph; p.pw = pw; p.dh = dh; p.dw = dw; p.pad_replicate = replicate;
  return *this;
}

PPConvCall& PPConvCall::out(__half* ptr, int cs, int co, int gstep) {
  p.out = ptr; p.out_cstride = cs; p.out_coff = co; p.out_fp32 = 0; p.out_gstep = gstep;
  return *this;
}

PPConvCall& PPConvCall::out_f32(float* ptr, int cs, int co) {
  p.out = ptr; p.out_cstride = cs; p.out_coff = co; p.out_fp32 = 1; p.out_gstep = 0;
  return *this;
}

PPConvCall& PPConvCall::act(int act1, float slope, float scale, int act2) {
  p.act1 = act1; p.slope = slope; p.scale = scale; p.act2 = act2;
  return *this;
}

PPConvCall& PPConvCall::residual(const __half* ptr, int cs, int co) {
  p.aux0 = ptr; p.aux0_cstride = cs; p.aux0_coff = co;
  return *this;
}

PPConvCall& PPConvCall::gru_zr(const __half* h, int h_cs, int h_co, __half* rh, int rh_cs, int rh_co) {
  p.epi = PP_EPI_GRU_ZR;
  p.aux0 = h; p.aux0_cstride = h_cs; p.aux0_coff = h_co;
  p.out2 = rh; p.out2_cstride = rh_cs; p.out2_coff = rh_co;
  return *this;
}

PPConvCall& PPConvCall::gru_h(const __half* h, int h_cs, int h_co, const __half* z, int z_cs, int z_co) {
  p.epi = PP_EPI_GRU_H;
  p.aux0 = h; p.aux0_cstride = h_cs; p.aux0_coff = h_co;
  p.aux1 = z; p.aux1_cstride = z_cs; p.aux1_coff = z_co;
  return *this;
}

PPConvCall& PPConvCall::in(const float* ptr, int C, int co, int channels) {
  if (err != PP_OK) return *this;
  if (n_split_in >= PP_MAX_SEGS / 3) {
    pp_set_error("conv %s: more than %d split-tf32 inputs", name.c_str(), PP_MAX_SEGS / 3);
    err = PP_ERR_ARG;
    return *this;
  }
  p.split = 1;
  split_in[n_split_in++] = SplitIn{ptr, C, co, channels};
  return *this;
}

PPConvCall& PPConvCall::out(float* ptr, int C, int co) {
  p.out = ptr; p.out_cstride = 2 * C; p.out_coff = co; p.out_lo = C; p.out_fp32 = 0; p.out_gstep = 0;
  return *this;
}

PPConvCall& PPConvCall::residual(const float* ptr, int C, int co) {
  p.aux0 = reinterpret_cast<const __half*>(ptr); p.aux0_cstride = 2 * C; p.aux0_coff = co; p.aux0_lo = C;
  return *this;
}

PPConvCall& PPConvCall::gru_zr(const float* h, int h_C, int h_co, float* rh, int rh_C, int rh_co) {
  p.epi = PP_EPI_GRU_ZR;
  p.aux0 = reinterpret_cast<const __half*>(h); p.aux0_cstride = 2 * h_C; p.aux0_coff = h_co; p.aux0_lo = h_C;
  p.out2 = reinterpret_cast<__half*>(rh); p.out2_cstride = 2 * rh_C; p.out2_coff = rh_co; p.out2_lo = rh_C;
  return *this;
}

PPConvCall& PPConvCall::gru_h(const float* h, int h_C, int h_co, const float* z, int z_C, int z_co) {
  p.epi = PP_EPI_GRU_H;
  p.aux0 = reinterpret_cast<const __half*>(h); p.aux0_cstride = 2 * h_C; p.aux0_coff = h_co; p.aux0_lo = h_C;
  p.aux1 = reinterpret_cast<const __half*>(z); p.aux1_cstride = 2 * z_C; p.aux1_coff = z_co; p.aux1_lo = z_C;
  return *this;
}

int PPConvCall::run(cudaStream_t st) {
  if (err != PP_OK) return err;
  if (p.split) {
    // (hi, lo, hi) passes over the inputs, in the kernel's 2-byte units: an fp32 channel is two of them
    PP_REQUIRE(p.nseg == 0 && n_split_in > 0, "conv %s: split-tf32 (float*) and fp16 inputs cannot be mixed", name.c_str());
    for (int pass = 0; pass < 3; ++pass)
      for (int i = 0; i < n_split_in; ++i) {
        const SplitIn& s = split_in[i];
        in(reinterpret_cast<const __half*>(s.ptr), 4 * s.C, 2 * (s.co + (pass == 1 ? s.C : 0)), 2 * s.channels);
      }
    if (err != PP_OK) return err;
  } else if (p.nseg > 0 && p.seg[p.nseg - 1].cend < p.Cin && p.Cin % 64 == 0 && p.Cin - p.seg[p.nseg - 1].cend < 64 &&
      p.seg[p.nseg - 1].gstep == 0) {
    // weights registered with their input channels zero-padded to a 64 multiple (engine.py PAD64_CONVS): the last
    // segment's tensor only holds `cvalid` channels, the TMA loads of the halo kernel zero-fill the rest
    PPConvSeg& last = p.seg[p.nseg - 1];
    last.cvalid = last.cend - last.cbegin;
    last.cend = p.Cin;
  }
  PP_REQUIRE(p.nseg > 0 && p.seg[p.nseg - 1].cend == p.Cin,
             "conv: input segments cover %d channels, weights expect %d", p.nseg ? p.seg[p.nseg - 1].cend : 0, p.Cin);
  PP_REQUIRE(p.out != nullptr, "conv: no output set");
  p.OH = (p.H + 2 * p.ph - p.dh * (p.kh - 1) - 1) / p.sh + 1;
  p.OW = (p.W + 2 * p.pw - p.dw * (p.kw - 1) - 1) / p.sw + 1;
  const double rows = (double)p.N * p.OH * p.OW;
  if (pp_prog_recording()) {     // part of a multi-layer program: recorded now, launched by pp_prog_end
    auto it = eng->convs.find(name);
    const double m = (it != eng->convs.end() && it->second.macs_per_pixel > 0.0) ? it->second.macs_per_pixel
                                                                                 : (double)p.Cout_g * p.groups * p.kh * p.kw * p.Cin;
    eng->prog_flops += 2.0 * rows * m;
    return pp_launch_conv(p, st);
  }
  eng->launches++;
  double macs = (double)p.Cout_g * p.groups * p.kh * p.kw * p.Cin;
  if (eng->profile) {
    auto it = eng->convs.find(name);
    if (it != eng->convs.end() && it->second.macs_per_pixel > 0.0) macs = it->second.macs_per_pixel;
  }
  PPProfScope ps(*eng, "conv:" + name, rows, 2.0 * rows * macs, 0.0, st);
  const int rc = pp_launch_conv(p, st);
  if (eng->profile && !eng->prof.empty())      // label the record with the kernel the launch was dispatched to
    eng->prof.back().name = std::string(pp_last_conv_kind() == 'g'   ? "conv:gemm:"
                                        : pp_last_conv_kind() == 'h' ? "conv:halo:"
                                                                     : "conv:igemm:") +
                            name;
  return rc;
}

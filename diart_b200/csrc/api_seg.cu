// Segmentation model handle (dg_seg_*) and the SincNet front end that both networks share.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <vector>

#include "host.cuh"

namespace dg {

// ParamSincFB.filters() in float32, as asteroid-filterbanks computes it with torch (SURVEY.md A.1)
static void sinc_filters(const float* low_hz_, const float* band_hz_, std::vector<float>& filt /*[251][80]*/) {
  filt.assign(251 * 80, 0.f);
  float n_[125], win[125];
  for (int i = 0; i < 125; i++) {
    const float t = (float)(i - 125) / 16000.0f;
    n_[i] = 6.283185307179586f * t;
    win[i] = (float)(0.54 - 0.46 * cos(2.0 * M_PI * i / 250.0));
  }
  for (int f = 0; f < 40; f++) {
    const float low = 50.f + fabsf(low_hz_[f]);
    float high = low + 50.f + fabsf(band_hz_[f]);
    high = fminf(fmaxf(high, 50.f), 8000.f);
    const float band = high - low, two_band = 2.f * band;
    for (int i = 0; i < 125; i++) {
      const float ft_low = low * n_[i], ft_high = high * n_[i], half_n = n_[i] / 2.f;
      const float lc = ((sinf(ft_high) - sinf(ft_low)) / half_n) * win[i];
      const float ls = ((cosf(ft_low) - cosf(ft_high)) / half_n) * win[i];
      filt[i * 80 + f] = lc / two_band;
      filt[(250 - i) * 80 + f] = lc / two_band;
      filt[i * 80 + 40 + f] = ls / two_band;
      filt[(250 - i) * 80 + 40 + f] = (-ls) / two_band;
    }
    filt[125 * 80 + f] = two_band / two_band;
    filt[125 * 80 + 40 + f] = 0.f / two_band;
  }
}

int prep_sincnet(const Tensors& t, const std::string& pre, SincWeights& w) {
  const float *g, *b;
  if (!(g = t.get(pre + "wav_norm1d.weight", 1)) || !(b = t.get(pre + "wav_norm1d.bias", 1))) return DG_EWEIGHT;
  w.wn_gamma = g[0];
  w.wn_beta = b[0];
  const float* lo = t.get(pre + "conv1d.0.filterbank.low_hz_", 40);
  const float* bd = t.get(pre + "conv1d.0.filterbank.band_hz_", 40);
  if (!lo || !bd) return DG_EWEIGHT;
  std::vector<float> h;
  sinc_filters(lo, bd, h);
  {
    std::vector<uint16_t> fp(2 * 80 * 256);
    sinc_tc_pack_filters(h.data(), fp.data());
    if (upload_u16(w.filt_planes, fp)) return DG_ECUDA;
    std::vector<float> cf(80);
    sinc_tc_affine_consts(h.data(), w.wn_beta, cf.data());
    if (upload(w.cf, cf)) return DG_ECUDA;
    std::vector<float> hs(80);
    sinc_tc_affine_consts(h.data(), 1.f, hs.data());
    if (upload(w.hsum, hs)) return DG_ECUDA;
  }
  auto pad_vec = [&](const std::string& name, int n, int npad, DevBuf& dst) -> int {
    const float* s = t.get(name, n);
    if (!s) return DG_EWEIGHT;
    std::vector<float> v(npad, 0.f);
    memcpy(v.data(), s, n * sizeof(float));
    return upload(dst, v) ? DG_ECUDA : 0;
  };
  int rc;
  if ((rc = pad_vec(pre + "norm1d.0.weight", 80, 80, w.g0)) || (rc = pad_vec(pre + "norm1d.0.bias", 80, 80, w.b0)) ||
      (rc = pad_vec(pre + "norm1d.1.weight", 60, 64, w.g1)) || (rc = pad_vec(pre + "norm1d.1.bias", 60, 64, w.b1)) ||
      (rc = pad_vec(pre + "norm1d.2.weight", 60, 64, w.g2)) || (rc = pad_vec(pre + "norm1d.2.bias", 60, 64, w.b2)) ||
      (rc = pad_vec(pre + "conv1d.1.bias", 60, 64, w.bias1)) || (rc = pad_vec(pre + "conv1d.2.bias", 60, 64, w.bias2)))
    return rc;
  auto conv_w_tc = [&](const std::string& name, int out, int in, int k, int in_pad, WeightPlanes& dst) -> int {
    const float* s = t.get(name, (int64_t)out * in * k);
    if (!s) return DG_EWEIGHT;
    std::vector<float> w_nk((size_t)out * k * in_pad, 0.f);
    for (int o = 0; o < out; o++)
      for (int c = 0; c < in; c++)
        for (int j = 0; j < k; j++) w_nk[(size_t)o * k * in_pad + j * in_pad + c] = s[((size_t)o * in + c) * k + j];
    return upload_split(dst, w_nk, out, 64, k * in_pad);
  };
  {
    // Conv1d(80, 60, 5) over 80-channel rows: K = 5 taps x 80 channels (the GEMM's halo mode)
    const float* s1 = t.get(pre + "conv1d.1.weight", (int64_t)60 * 80 * 5);
    if (!s1) return DG_EWEIGHT;
    std::vector<float> w_nk((size_t)60 * 400, 0.f);
    for (int o = 0; o < 60; o++)
      for (int c = 0; c < 80; c++)
        for (int j = 0; j < 5; j++) w_nk[(size_t)o * 400 + j * 80 + c] = s1[((size_t)o * 80 + c) * 5 + j];
    if (upload_split(w.w1, w_nk, 60, 64, 400)) return DG_ECUDA;
  }
  if ((rc = conv_w_tc(pre + "conv1d.2.weight", 60, 60, 5, 64, w.w2))) return rc;
  return 0;
}


int run_sinc_prep(SincPrep& p, const float* wav, int B, const Geom& g, cudaStream_t st, int hop,
                  bool overlap_known) {
  int rc;
  if ((rc = p.ensure(B, g))) return rc;
  // stream form of the sinc layer: only with a hop hint from the caller; the device flag written by overlap_check
  // decides per batch, so a wrong hint costs a few empty launches, never a wrong result
  p.hop = 0;
  if (hop > 0 && B >= 4 && hop % 40 == 0 && g.S % 4 == 0 && hop < g.S && ((uintptr_t)wav & 15) == 0) {
    if ((rc = p.ensure_stream(B, g, hop))) return rc;
    if (overlap_known) {   // the batch was formed on the device from ONE stream (dg_stream): nothing to verify
      DG_CUDA(cudaMemsetAsync(p.flag.p, 1, sizeof(int), st));
    } else if ((rc = launch_overlap_check(wav, B, g.S, hop, p.flag.as<int>(), st))) {
      return rc;
    }
    p.hop = hop;
  }
  const bool fast_stats = p.hop && stream_stats_ok(g.S, p.hop);
  if (fast_stats) {
    if (p.spart.ensure(stream_stats_doubles(B, g.S, p.hop) * 8)) return DG_ECUDA;
    if ((rc = launch_stream_stats(wav, B, g.S, p.hop, p.spart.as<double>(), p.wmean.as<float>(), p.wrstd.as<float>(),
                                  p.flag.as<int>(), st)))
      return rc;
  }
  if ((rc = launch_wave_stats(wav, B, g.S, p.wmean.as<float>(), p.wrstd.as<float>(), st, fast_stats ? p.flag.as<int>() : nullptr)))
    return rc;
  if (p.hop && (rc = launch_stream_prep(wav, p.wrstd.as<float>(), B, g, hop, p.swh.p, p.swl.p, p.flag.as<int>(), st))) return rc;
  return launch_sinc_prep(wav, p.wmean.as<float>(), p.wrstd.as<float>(), B, g, p.wh.p, p.wl.p, st,
                          p.hop ? p.flag.as<int>() : nullptr);
}

// waveform [B,S] -> k.out (pre-norm conv2 output, pooled [B*S2,64] or un-pooled [B*S1,64]) + its
// InstanceNorm scale/shift (k.sc2, k.sh2)
int run_sincnet(const SincWeights& w, SincWork& k, const float* wav, int B, const Geom& g, cudaStream_t st,
                const SincPrep* shared) {
  int rc;
  if ((rc = k.ensure(B, g))) return rc;
  const int* stream_flag = nullptr;      // device flag "the stream form produced the conv1 operand planes of this batch"
  const SincPrep* prep = shared;
  if (!prep) {
    if ((rc = run_sinc_prep(k.own_prep, wav, B, g, st))) return rc;
    prep = &k.own_prep;
  }
  if (prep->hop) {   // stream form: one convolution of the unique samples + a per-window affine / |.| / pool pass
    const SincStreamGeom sg = sinc_stream_geom(B, g, prep->hop);
    if (k.craw.ensure(((size_t)sg.P + 16) * 80 * 4) || k.part.ensure(sinc_pool_part_floats(B, g, prep->hop) * 4)) return DG_ECUDA;
    // raw convolution of the stream, then statistics and normalised operand planes straight from it (p0 is never written)
    if ((rc = launch_sinc0_tc_stream(w.filt_planes.p, B, g, prep->hop, prep->swh.p, prep->swl.p, k.craw.as<float>(),
                                     prep->flag.as<int>(), st)) ||
        (rc = launch_sinc_pool_fused(k.craw.as<float>(), prep->wmean.as<float>(), prep->wrstd.as<float>(), w.cf.as<float>(),
                                     w.hsum.as<float>(), w.wn_gamma, B, g, prep->hop, w.g0.as<float>(), w.b0.as<float>(),
                                     k.part.as<float>(), k.sc0.as<float>(), k.sh0.as<float>(), k.a0h.p, k.a0l.p,
                                     prep->flag.as<int>(), st)))
      return rc;
    stream_flag = prep->flag.as<int>();
  }
  if ((rc = launch_sinc0_tc(w.wn_gamma, w.cf.as<float>(), w.filt_planes.p, B, g, prep->wh.p, prep->wl.p, k.p0.as<float>(), st,
                            stream_flag)))
    return rc;
  if ((rc = launch_instnorm_stats(k.p0.as<float>(), B, g.S0, g.T0, 80, 80, w.g0.as<float>(), w.b0.as<float>(),
                                  k.sc0.as<float>(), k.sh0.as<float>(), st, 0, stream_flag)))
    return rc;
  // Conv1d(80,60,5): normalised input as fp16 hi/lo planes (80-channel rows)
  const long long M0 = (long long)B * g.S0, M1 = (long long)B * g.S1;
  if ((rc = launch_split_ex(k.p0.as<float>(), M0, 80, 80, 80, 0, g.S0, k.sc0.as<float>(), k.sh0.as<float>(),
                            k.a0h.p, k.a0l.p, st, stream_flag)))
    return rc;
  // conv1 / conv2 with MaxPool1d(3) and the InstanceNorm partial sums in the GEMM epilogue (TC_MAXPOOL3): the un-pooled maps are
  // never written, the statistics pass reads 2 x 3 x 64 floats per tile.  Needs a tile of 96..126 rows that divides the item at both
  // stages; otherwise the un-pooled float32 map -> instnorm_stats -> split with pooling on load
  const int tr0 = gemm_tc_pool3_tile_rows(g.S0), tr1 = gemm_tc_pool3_tile_rows(g.S1);
  if (tr0 && tr1) {
    if (k.part3.ensure((size_t)(M0 / tr0) * 2 * TC_POOL3_SLOTS * 64 * 4)) return DG_ECUDA;
    TcGemm t{};
    t.A_hi = k.a0h.p; t.A_lo = k.a0l.p; t.lda = 80; t.Cin = 80; t.KW = 5; t.dil = 1; t.Mtot = M0; t.M = M0;
    t.N = 64; t.bias = w.bias1.as<float>(); t.out_f32 = k.p1.as<float>(); t.ldc = 64; t.epi = 5; t.tag = "sinc_conv1";
    t.pool_part = k.part3.as<float>(); t.pool_item_rows = g.S0; t.pool3_T = g.T1; t.pool3_tile_rows = tr0;
    if ((rc = set_weights(t, w.w1)) || (rc = launch_gemm_tc(t, st)) ||
        (rc = launch_instnorm_finalize(k.part3.as<float>(), B, g.S0, tr0, g.T1, 64, 64, w.bias1.as<float>(), w.g1.as<float>(),
                                       w.b1.as<float>(), k.sc1.as<float>(), k.sh1.as<float>(), 64, st)) ||
        (rc = launch_split_ex(k.p1.as<float>(), M1, 64, 64, 64, 0, g.S1, k.sc1.as<float>(), k.sh1.as<float>(), k.a1h.p, k.a1l.p, st)))
      return rc;
    t.A_hi = k.a1h.p; t.A_lo = k.a1l.p; t.lda = 64; t.Cin = 64; t.KW = 5; t.Mtot = M1; t.M = M1;
    t.bias = w.bias2.as<float>(); t.out_f32 = k.p2.as<float>(); t.tag = "sinc_conv2";
    t.pool_item_rows = g.S1; t.pool3_T = g.T2; t.pool3_tile_rows = tr1;
    if ((rc = set_weights(t, w.w2)) || (rc = launch_gemm_tc(t, st))) return rc;
    k.out = k.p2.as<float>();
    k.out_pool = 0;
    return launch_instnorm_finalize(k.part3.as<float>(), B, g.S1, tr1, g.T2, 64, 64, w.bias2.as<float>(), w.g2.as<float>(),
                                    w.b2.as<float>(), k.sc2.as<float>(), k.sh2.as<float>(), 64, st);
  }
  TcGemm t{};
  t.A_hi = k.a0h.p; t.A_lo = k.a0l.p; t.lda = 80; t.Cin = 80; t.KW = 5; t.dil = 1; t.Mtot = M0; t.M = M0;
  t.N = 64; t.bias = w.bias1.as<float>(); t.out_f32 = k.c1.as<float>(); t.ldc = 64; t.epi = 0; t.tag = "sinc_conv1";
  if ((rc = set_weights(t, w.w1)) || (rc = launch_gemm_tc(t, st))) return rc;
  if ((rc = launch_instnorm_stats(k.c1.as<float>(), B, g.S0, g.T1, 64, 64, w.g1.as<float>(), w.b1.as<float>(),
                                  k.sc1.as<float>(), k.sh1.as<float>(), st, 1)))
    return rc;
  // Conv1d(60,60,5) on MaxPool(conv1) -> norm -> leaky, again un-pooled output
  if ((rc = launch_split_ex(k.c1.as<float>(), M1, 64, 64, 64, 1, g.S1, k.sc1.as<float>(), k.sh1.as<float>(),
                            k.a1h.p, k.a1l.p, st)))
    return rc;
  t.A_hi = k.a1h.p; t.A_lo = k.a1l.p; t.lda = 64; t.Cin = 64; t.KW = 5; t.Mtot = M1; t.M = M1;
  t.bias = w.bias2.as<float>(); t.out_f32 = k.c2.as<float>(); t.tag = "sinc_conv2";
  if ((rc = set_weights(t, w.w2)) || (rc = launch_gemm_tc(t, st))) return rc;
  k.out = k.c2.as<float>();
  k.out_pool = 1;
  return launch_instnorm_stats(k.c2.as<float>(), B, g.S1, g.T2, 64, 64, w.g2.as<float>(), w.b2.as<float>(),
                               k.sc2.as<float>(), k.sh2.as<float>(), st, 1);
}

int debug_copy_map(const char* who, const void* hi, const void* lo, int B, int item_rows, int ld, int T, int C, float* out_host,
                   int64_t cap, int* dims) {
  dims[0] = B; dims[1] = T; dims[2] = C;
  if ((int64_t)B * T * C > cap) {
    set_error(std::string(who) + ": buffer too small");
    return DG_EINVAL;
  }
  const size_t n = (size_t)B * item_rows * ld;
  std::vector<float> full(n);
  if (lo) {
    std::vector<uint16_t> vh(n), vl(n);
    DG_CUDA(cudaMemcpy(vh.data(), hi, n * 2, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(vl.data(), lo, n * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; i++) full[i] = host_h16_to_f32(vh[i]) + host_h16_to_f32(vl[i]);
  } else {
    DG_CUDA(cudaMemcpy(full.data(), hi, n * 4, cudaMemcpyDeviceToHost));
  }
  for (int b = 0; b < B; b++)
    for (int t = 0; t < T; t++)
      memcpy(out_host + ((size_t)b * T + t) * C, &full[((size_t)b * item_rows + t) * ld], (size_t)C * 4);
  return DG_OK;
}

int debug_copy_front(const char* who, int stage, const SincWork& k, const SincPrep* prep, const void* xh, const void* xl, int B,
                     const Geom& g, float* out_host, int64_t cap, int* dims) {
  if (stage == 0) return debug_copy_map(who, k.a0h.p, k.a0l.p, B, g.S0, 80, g.T0, 80, out_host, cap, dims);
  if (stage == 1) return debug_copy_map(who, k.a1h.p, k.a1l.p, B, g.S1, 64, g.T1, 60, out_host, cap, dims);
  if (stage == 2) return debug_copy_map(who, xh, xl, B, g.S2, 64, g.T2, 60, out_host, cap, dims);
  const SincPrep& p = prep ? *prep : k.own_prep;
  dims[0] = 2; dims[1] = B; dims[2] = 1;
  if (2 * B > cap) {
    set_error(std::string(who) + ": buffer too small");
    return DG_EINVAL;
  }
  DG_CUDA(cudaMemcpy(out_host, p.wmean.p, (size_t)B * 4, cudaMemcpyDeviceToHost));
  DG_CUDA(cudaMemcpy(out_host + B, p.wrstd.p, (size_t)B * 4, cudaMemcpyDeviceToHost));
  return DG_OK;
}

int debug_front_paths(const SincPrep* prep, const Geom& g, int* paths) {
  *paths = 0;
  if (prep && prep->hop) {
    int flag = 0;
    DG_CUDA(cudaMemcpy(&flag, prep->flag.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag) *paths |= DG_DBG_STREAM_FORM;
  }
  if (gemm_tc_pool3_tile_rows(g.S0) && gemm_tc_pool3_tile_rows(g.S1)) *paths |= DG_DBG_POOL3_FUSED;
  return DG_OK;
}

}  // namespace dg

extern "C" int dg_selftest_sinc_filters_host(const float* low_hz, const float* band_hz, float* filters) {
  if (!low_hz || !band_hz || !filters) {
    set_error("dg_selftest_sinc_filters_host: null argument");
    return DG_EINVAL;
  }
  std::vector<float> h;
  sinc_filters(low_hz, band_hz, h);
  memcpy(filters, h.data(), h.size() * sizeof(float));
  return DG_OK;
}

static int seg_prepare(dg_seg* h, const Tensors& t) {
  int rc;
  if ((rc = prep_sincnet(t, "sincnet.", h->sw))) return rc;
  for (int L = 0; L < 4; L++) {
    const int in = L == 0 ? 60 : 256, in_pad = L == 0 ? 64 : 256;
    // gate rows n = direction * 512 + r of both directions, input channels padded to in_pad
    std::vector<float> w_nk((size_t)1024 * in_pad, 0.f), b(1024, 0.f);
    const float* hh[2];
    for (int d = 0; d < 2; d++) {
      const std::string sfx = "_l" + std::to_string(L) + (d ? "_reverse" : "");
      const float* wi = t.get("lstm.weight_ih" + sfx, (int64_t)512 * in);
      const float* bi = t.get("lstm.bias_ih" + sfx, 512);
      const float* bh = t.get("lstm.bias_hh" + sfx, 512);
      hh[d] = t.get("lstm.weight_hh" + sfx, 512 * 128);
      if (!wi || !bi || !bh || !hh[d]) return DG_EWEIGHT;
      for (int r = 0; r < 512; r++) {
        for (int c = 0; c < in; c++) w_nk[(size_t)(d * 512 + r) * in_pad + c] = wi[(size_t)r * in + c];
        b[d * 512 + r] = bi[r] + bh[r];
      }
    }
    if (upload(h->bih[L], b) || upload_split(h->wih[L], w_nk, 1024, 1024, in_pad)) return DG_ECUDA;
    {
      std::vector<uint16_t> rh(lstm_tc_plane_elems()), rl(lstm_tc_plane_elems());
      h->whh[L].scale = lstm_tc_pack_whh(hh[0], hh[1], rh.data(), rl.data());
      if (upload_u16(h->whh[L].hi, rh) || upload_u16(h->whh[L].lo, rl)) return DG_ECUDA;
    }
  }
  {
    const float* w0 = t.get("linear.0.weight", 128 * 256);
    const float* b0 = t.get("linear.0.bias", 128);
    const float* w1 = t.get("linear.1.weight", 128 * 128);
    const float* b1 = t.get("linear.1.bias", 128);
    if (!w0 || !b0 || !w1 || !b1) return DG_EWEIGHT;
    if (upload(h->l1b, std::vector<float>(b0, b0 + 128)) || upload(h->l2b, std::vector<float>(b1, b1 + 128)) ||
        upload_split(h->l1, std::vector<float>(w0, w0 + 128 * 256), 128, 128, 256) ||
        upload_split(h->l2, std::vector<float>(w1, w1 + 128 * 128), 128, 128, 128) ||
        upload(h->ones128, std::vector<float>(128, 1.f)) || upload(h->zeros128, std::vector<float>(128, 0.f)))
      return DG_ECUDA;
  }
  const int64_t cn = t.numel("classifier.bias");
  if (cn < 1 || cn > 8) {
    set_error("classifier.bias missing or more than 8 local speakers");
    return DG_EWEIGHT;
  }
  h->K = (int)cn;
  const float* cw = t.get("classifier.weight", cn * 128);
  const float* cb = t.get("classifier.bias", cn);
  if (!cw || !cb) return DG_EWEIGHT;
  if (upload(h->cw, std::vector<float>(cw, cw + cn * 128)) || upload(h->cb, std::vector<float>(cb, cb + cn)))
    return DG_ECUDA;
  return 0;
}

extern "C" int dg_seg_create(const dg_tensor* tensors, int n, int device, dg_seg** out) {
  if (!tensors || !out) {
    set_error("dg_seg_create: null argument");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_seg> h(new dg_seg());
  h->device = device;
  Tensors t(tensors, n);
  int rc = seg_prepare(h.get(), t);
  if (rc) return rc;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_seg_dims(const dg_seg* h, int num_samples, int* frames, int* speakers) {
  if (!h || num_samples < 3000) {
    set_error("dg_seg_dims: bad arguments");
    return DG_EINVAL;
  }
  Geom g = make_geom(num_samples);
  if (frames) *frames = g.T2;
  if (speakers) *speakers = h->ps_speakers ? h->ps_speakers : h->K;
  return DG_OK;
}

// Declares the model a powerset model (pyannote/segmentation-3.0 style): its classifier has one output per subset of
// the `num_speakers` local speakers of size <= `max_per_frame`, in itertools.combinations order (pyannote
// Powerset.build_mapping); the forward then returns hard multilabel scores (reference models.py:29-39).
extern "C" int dg_seg_set_powerset(dg_seg* h, int num_speakers, int max_per_frame) {
  if (!h || num_speakers < 1 || num_speakers > 8 || max_per_frame < 0 || max_per_frame > num_speakers) {
    set_error("dg_seg_set_powerset: bad arguments");
    return DG_EINVAL;
  }
  std::vector<uint32_t> masks;
  for (int size = 0; size <= max_per_frame; size++)          // subsets by size, each size in lexicographic order
    for (uint32_t m = 0; m < (1u << num_speakers); m++) {
      if (__builtin_popcount(m) != size) continue;
      masks.push_back(m);
    }
  // lexicographic order of combinations (0,1) < (0,2) < (1,2) is NOT numeric order of the bit masks in general: sort each
  // size class by the sorted member tuples
  auto members = [&](uint32_t m) {
    std::vector<int> v;
    for (int i = 0; i < num_speakers; i++)
      if (m >> i & 1u) v.push_back(i);
    return v;
  };
  std::stable_sort(masks.begin(), masks.end(), [&](uint32_t a, uint32_t b) {
    const int sa = __builtin_popcount(a), sb = __builtin_popcount(b);
    if (sa != sb) return sa < sb;
    return members(a) < members(b);
  });
  if ((int)masks.size() != h->K) {
    set_error("dg_seg_set_powerset: the classifier has " + std::to_string(h->K) + " outputs but the powerset has " +
              std::to_string(masks.size()) + " classes");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  if (h->ps_masks.ensure(masks.size() * 4)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->ps_masks.p, masks.data(), masks.size() * 4, cudaMemcpyHostToDevice));
  h->ps_speakers = num_speakers;
  return DG_OK;
}

// classifier + sigmoid, or classifier + powerset decoding
static int seg_head_final(dg_seg* h, const float* y2, int B, const Geom& g, float* seg, cudaStream_t st) {
  if (h->ps_speakers)
    return launch_seg_powerset(y2, h->cw.as<float>(), h->cb.as<float>(), B, g.T2, g.S2, h->K, h->ps_speakers,
                               h->ps_masks.as<unsigned>(), seg, st);
  return launch_seg_final(y2, h->cw.as<float>(), h->cb.as<float>(), B, g.T2, g.S2, h->K, seg, st);
}

int seg_forward_lane(dg_seg* h, int lane, const SincPrep* prep, const float* wav, int B, int S, float* seg,
                     cudaStream_t st, int stop_after) {
  DG_CUDA(cudaSetDevice(h->device));
  dg_seg::Scratch& w = h->scr[lane];
  const Geom g = make_geom(S);
  int rc;
  if ((rc = run_sincnet(h->sw, w.work, wav, B, g, st, prep))) return rc;
  const size_t rows = (size_t)B * g.S2 + 64;
  if (w.gx.ensure(rows * 1024 * 4) || w.y2.ensure(rows * 128 * 4) || w.xh.ensure(rows * 256 * 2) ||
      w.xl.ensure(rows * 256 * 2) || w.y1h.ensure(rows * 128 * 2) || w.y1l.ensure(rows * 128 * 2))
    return DG_ECUDA;
  const long long M = (long long)B * g.S2;
  if ((rc = launch_split_ex(w.work.out, M, 64, 64, 64, w.work.out_pool, g.S2, w.work.sc2.as<float>(), w.work.sh2.as<float>(),
                            w.xh.p, w.xl.p, st)))
    return rc;
  for (int L = 0; L < 4 && L <= stop_after; L++) {
    const int cin = L == 0 ? 64 : 256;
    TcGemm t{};
    t.A_hi = w.xh.p; t.A_lo = w.xl.p; t.lda = cin; t.Cin = cin; t.KW = 1; t.dil = 1; t.Mtot = M; t.M = M;
    t.N = 1024; t.bias = h->bih[L].as<float>(); t.out_f32 = w.gx.as<float>(); t.ldc = 1024; t.epi = 0; t.tag = "lstm_inproj";
    if ((rc = set_weights(t, h->wih[L])) || (rc = launch_gemm_tc(t, st))) return rc;
    // the recurrence writes h_t straight into the operand planes of the next GEMM (the in-projection that read them has
    // completed in stream order)
    if ((rc = launch_lstm_layer_tc(w.gx.as<float>(), h->whh[L].hi.p, h->whh[L].lo.p, h->whh[L].scale, B, g.T2, g.S2, nullptr,
                                   w.xh.p, w.xl.p, st)))
      return rc;
  }
  if (stop_after < 3) return 0;
  // Linear(256,128) -> leaky -> Linear(128,128) -> leaky on the tensor-core GEMM (identity "BatchNorm")
  TcGemm t{};
  t.A_hi = w.xh.p; t.A_lo = w.xl.p; t.lda = 256; t.Cin = 256; t.KW = 1; t.dil = 1; t.Mtot = M; t.M = M;
  t.N = 128; t.bias = h->l1b.as<float>(); t.bn_scale = h->ones128.as<float>(); t.bn_shift = h->zeros128.as<float>();
  t.out_hi = w.y1h.p; t.out_lo = w.y1l.p; t.ldc = 128; t.epi = 1; t.tag = "seg_linear";
  if ((rc = set_weights(t, h->l1)) || (rc = launch_gemm_tc(t, st))) return rc;
  t.A_hi = w.y1h.p; t.A_lo = w.y1l.p; t.lda = 128; t.Cin = 128; t.bias = h->l2b.as<float>();
  t.out_hi = nullptr; t.out_lo = nullptr; t.out_f32 = w.y2.as<float>(); t.epi = 2;
  if ((rc = set_weights(t, h->l2)) || (rc = launch_gemm_tc(t, st))) return rc;
  return seg_head_final(h, w.y2.as<float>(), B, g, seg, st);
}

extern "C" int dg_seg_forward(dg_seg* h, const float* wav, int B, int S, float* seg, void* stream) {
  if (!h || !wav || !seg || B < 1 || S < 3000) {
    set_error("dg_seg_forward: bad arguments (need B >= 1, S >= 3000)");
    return DG_EINVAL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  DG_CUDA(cudaSetDevice(h->device));
  LaneUse use(h->guard[0], stream ? stream : (void*)h, st);
  int rc;
  if ((rc = use.rc) || (rc = seg_forward_lane(h, 0, nullptr, wav, B, S, seg, st))) return rc;
  return use.end();
}

// test hook: the production forward (run_sinc_prep with the hop hint as dg_pipeline_set_hop gives it, seg_forward_lane) with a
// host-side stop point, and one intermediate map copied to the host
extern "C" int dg_seg_debug_stage(dg_seg* h, const float* wav_dev, int B, int S, int hop, int stage, float* out_host, int64_t cap,
                                  int* dims) {
  if (!h || !wav_dev || !out_host || !dims || B < 1 || S < 3000 || hop < 0 || stage < 0 || stage > 10) {
    set_error("dg_seg_debug_stage: bad arguments (need a segmentation handle, B >= 1, S >= 3000, stage 0..10)");
    return DG_EINVAL;
  }
  const int speakers = h->ps_speakers ? h->ps_speakers : h->K;     // columns of the scores (powerset: decoded labels)
  DG_CUDA(cudaSetDevice(h->device));
  const Geom g = make_geom(S);
  const char* who = "dg_seg_debug_stage";
  cudaStream_t st = nullptr;
  SincPrep shared;
  const SincPrep* prep = nullptr;
  DevBuf seg;
  int rc;
  if (seg.ensure((size_t)B * g.T2 * speakers * 4)) return DG_ECUDA;
  {
    LaneUse use(h->guard[0], h, st);
    if ((rc = use.rc)) return rc;
    if (hop > 0) {
      if ((rc = run_sinc_prep(shared, wav_dev, B, g, st, hop, false))) return rc;
      prep = &shared;
    }
    if ((rc = seg_forward_lane(h, 0, prep, wav_dev, B, S, seg.as<float>(), st, stage <= 3 ? -1 : stage <= 7 ? stage - 4 : 99)))
      return rc;
  }
  DG_CUDA(cudaDeviceSynchronize());
  if ((rc = debug_front_paths(prep, g, &dims[3]))) return rc;
  if (lstm_tc_rows(B) == 16) dims[3] |= DG_DBG_LSTM_16ROWS;
  const dg_seg::Scratch& w = h->scr[0];
  if (stage <= 3) return debug_copy_front(who, stage, w.work, prep, w.xh.p, w.xl.p, B, g, out_host, cap, dims);
  if (stage <= 7) return debug_copy_map(who, w.xh.p, w.xl.p, B, g.S2, 256, g.T2, 256, out_host, cap, dims);
  if (stage == 8) return debug_copy_map(who, w.y1h.p, w.y1l.p, B, g.S2, 128, g.T2, 128, out_host, cap, dims);
  if (stage == 9) return debug_copy_map(who, w.y2.p, nullptr, B, g.S2, 128, g.T2, 128, out_host, cap, dims);
  return debug_copy_map(who, seg.p, nullptr, B, g.T2, speakers, g.T2, speakers, out_host, cap, dims);
}

extern "C" int dg_seg_destroy(dg_seg* h) {
  delete h;
  return DG_OK;
}

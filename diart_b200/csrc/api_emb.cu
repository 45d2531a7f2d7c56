// Embedding model handle (dg_emb_*): the x-vector network and variant B (WeSpeaker ResNet34), and the element-wise blocks.
#include <math.h>
#include <string.h>

#include <memory>
#include <vector>

#include "host.cuh"

namespace dg {

int launch_stats_pool_ex(const float* x, int stride, int T, int C, const float* w, int F, int K, int layout,
                         int n_groups, const int* grp_item, const int* grp_q0, const int* grp_nq, const int* idx0,
                         const int* idx1, const float* lam1, float eps, float* pooled, cudaStream_t st,
                         long long item_pitch = 0, int row_pitch = 0);

}  // namespace dg

// ---- variant B: WeSpeaker ResNet34 (SURVEY.md 8(a) A8'; kernels in resnet.cu + the Conv2d epilogue of gemm_tc.cu)
struct ResConv {                       // Conv2d (3x3 pad 1 or 1x1, no bias) + folded BatchNorm2d(eval)
  int cin = 0, cout = 0, ksize = 3, stride = 1;
  int KW = 9, cin_gemm = 0, lda = 0;   // GEMM view: taps, channels consumed per tap, row pitch of the input planes
  WeightPlanes w;
  DevBuf sc, sh;
};
struct ResBlock {
  ResConv c1, c2, sc;
  bool has_sc = false;
};
struct ResNet {
  WeightPlanes fb;               // kaldi fbank frame operator [640][448]
  DevBuf banks, k_lo, k_hi, stem_w, stem_sc, stem_sh;
  std::vector<ResBlock> blocks;
  int stage_of[16];
  // work buffers: planes of the waveform, 1 / their scale per item and the level of its constant 80-sample pieces, spectrum,
  // log-mel map, three plane pairs per stage, float32 final map
  DevBuf wav_hi, wav_lo, inv_s, level, spec, logmel, mean, act[4][3][2], fin;
  int last_S = 0;                // the padding rings are only valid for one geometry: buffers are cleared when it changes
  int stop_after = 99;           // test hook (dg_emb_debug_trunk): stop after the stem (-1) / after block k
  int dbg_stage = 0, dbg_buf = 0;
};
static const int RN_CH[4] = {32, 64, 128, 256};
static const int RN_BLOCKS[4] = {3, 4, 6, 3};

static const int TD_OUT[5] = {512, 512, 512, 512, 1500};
static const int TD_K[5] = {5, 3, 3, 1, 1};
static const int TD_DIL[5] = {1, 2, 3, 1, 1};

static int resnet_prepare(dg_emb* h, const Tensors& t);

static int emb_prepare(dg_emb* h, const Tensors& t) {
  int rc;
  if (t.numel("resnet.conv1.weight") > 0) return resnet_prepare(h, t);     // variant B checkpoint
  if ((rc = prep_sincnet(t, "sincnet.", h->sw))) return rc;
  int in = 60, in_pad = 64;
  for (int L = 0; L < 5; L++) {
    const int out = TD_OUT[L], k = TD_K[L];
    const std::string cv = "tdnns." + std::to_string(3 * L), bn = "tdnns." + std::to_string(3 * L + 2);
    const float* w = t.get(cv + ".weight", (int64_t)out * in * k);
    const float* b = t.get(cv + ".bias", out);
    const float* gm = t.get(bn + ".weight", out);
    const float* bt = t.get(bn + ".bias", out);
    const float* rm = t.get(bn + ".running_mean", out);
    const float* rv = t.get(bn + ".running_var", out);
    if (!w || !b || !gm || !bt || !rm || !rv) return DG_EWEIGHT;
    std::vector<float> bv(b, b + out), sc(out), sf(out);
    for (int o = 0; o < out; o++) {
      // BatchNorm1d(eval): (x - mean) / sqrt(var + 1e-5) * gamma + beta  ==  x * sc + sf
      sc[o] = gm[o] / sqrtf(rv[o] + 1e-5f);
      sf[o] = bt[o] - rm[o] * sc[o];
    }
    if (upload(h->tb[L], bv) || upload(h->bns[L], sc) || upload(h->bnh[L], sf)) return DG_ECUDA;
    {
      const int K = k * in_pad, npad = (out + 255) / 256 * 256;
      std::vector<float> w_nk((size_t)out * K, 0.f);
      for (int o = 0; o < out; o++)
        for (int c = 0; c < in; c++)
          for (int j = 0; j < k; j++) w_nk[(size_t)o * K + j * in_pad + c] = w[((size_t)o * in + c) * k + j];
      if (upload_split(h->tw[L], w_nk, out, npad, K)) return DG_ECUDA;
    }
    in = out;
    in_pad = out;
  }
  const int64_t dn = t.numel("embedding.bias");
  if (dn < 4 || dn % 4) {
    set_error("embedding.bias missing or dimension not a multiple of 4");
    return DG_EWEIGHT;
  }
  h->D = (int)dn;
  const float* ew = t.get("embedding.weight", dn * 3000);
  const float* eb = t.get("embedding.bias", dn);
  if (!ew || !eb) return DG_EWEIGHT;
  if (upload(h->eb, std::vector<float>(eb, eb + dn))) return DG_ECUDA;
  {
    std::vector<float> w_nk((size_t)dn * 3008, 0.f);
    for (int o = 0; o < dn; o++) memcpy(&w_nk[(size_t)o * 3008], ew + (size_t)o * 3000, 3000 * sizeof(float));
    if (upload_split(h->ew, w_nk, (int)dn, ((int)dn + 255) / 256 * 256, 3008)) return DG_ECUDA;
  }
  return 0;
}

// Conv2d weight [co][ci][kh (mel)][kw (time)] + BatchNorm2d -> GEMM weight planes [Npad][K] (tap-major K) + scale / shift.
// Maps are [item][w = time][h = mel][C]: tap (dw, dh) multiplies w[co][ci][dh][dw].  With 32 input channels the three dh
// taps of one dw are 96 CONTIGUOUS values of the input planes (rows h-1, h, h+1 follow each other in memory), so they are
// read as one 128-wide K slab through an overlapping-row view (row pitch 32): 3 taps x 128 instead of 9 taps x 64.
static int resnet_conv_prepare(const Tensors& t, const std::string& conv, const std::string& bn, int cin, int cout, int ksize,
                               int stride, ResConv& c) {
  const float* w = t.get(conv + ".weight", (int64_t)cout * cin * ksize * ksize);
  const float* gm = t.get(bn + ".weight", cout);
  const float* bt = t.get(bn + ".bias", cout);
  const float* rm = t.get(bn + ".running_mean", cout);
  const float* rv = t.get(bn + ".running_var", cout);
  if (!w || !gm || !bt || !rm || !rv) return DG_EWEIGHT;
  c.cin = cin; c.cout = cout; c.ksize = ksize; c.stride = stride;
  const bool narrow = cin == 32;
  if (ksize == 3) {
    c.KW = narrow ? 3 : 9;
    c.cin_gemm = narrow ? 128 : cin;
  } else {
    c.KW = 1;
    c.cin_gemm = narrow ? 64 : cin;
  }
  c.lda = cin;
  const int K = c.KW * c.cin_gemm;
  const int npad = cout <= 64 ? cout : (cout + 127) / 128 * 128;
  std::vector<float> w_nk((size_t)cout * K, 0.f), sc(cout), sh(cout);
  for (int o = 0; o < cout; o++) {
    for (int ci = 0; ci < cin; ci++)
      for (int dh = 0; dh < ksize; dh++)
        for (int dw = 0; dw < ksize; dw++) {
          const float v = w[(((size_t)o * cin + ci) * ksize + dh) * ksize + dw];
          size_t k;
          if (ksize == 1) k = ci;
          else if (narrow) k = (size_t)dw * 128 + dh * 32 + ci;
          else k = (size_t)(dw * 3 + dh) * cin + ci;
          w_nk[(size_t)o * K + k] = v;
        }
    sc[o] = gm[o] / sqrtf(rv[o] + 1e-5f);
    sh[o] = bt[o] - rm[o] * sc[o];
  }
  if (upload_split(c.w, w_nk, cout, npad, K) || upload(c.sc, sc) || upload(c.sh, sh)) return DG_ECUDA;
  return 0;
}

static int resnet_prepare(dg_emb* h, const Tensors& t) {
  int rc;
  h->variant = 1;
  h->rn.reset(new ResNet());
  ResNet& r = *h->rn;
  {
    std::vector<float> op;
    fbank_frame_operator(op);                                   // [514][400]
    std::vector<float> w_nk((size_t)514 * 448, 0.f);
    for (int n = 0; n < 514; n++) memcpy(&w_nk[(size_t)n * 448], &op[(size_t)n * 400], 400 * sizeof(float));
    if (upload_split(r.fb, w_nk, 514, 640, 448)) return DG_ECUDA;
    std::vector<float> banks;
    std::vector<int> lo, hi;
    fbank_mel_banks(banks, lo, hi);
    if (upload(r.banks, banks) || r.k_lo.ensure(80 * 4) || r.k_hi.ensure(80 * 4)) return DG_ECUDA;
    DG_CUDA(cudaMemcpy(r.k_lo.p, lo.data(), 80 * 4, cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(r.k_hi.p, hi.data(), 80 * 4, cudaMemcpyHostToDevice));
  }
  {
    const float* w = t.get("resnet.conv1.weight", 32 * 9);
    const float* gm = t.get("resnet.bn1.weight", 32);
    const float* bt = t.get("resnet.bn1.bias", 32);
    const float* rm = t.get("resnet.bn1.running_mean", 32);
    const float* rv = t.get("resnet.bn1.running_var", 32);
    if (!w || !gm || !bt || !rm || !rv) return DG_EWEIGHT;
    std::vector<float> sc(32), sh(32);
    for (int o = 0; o < 32; o++) {
      sc[o] = gm[o] / sqrtf(rv[o] + 1e-5f);
      sh[o] = bt[o] - rm[o] * sc[o];
    }
    if (upload(r.stem_w, std::vector<float>(w, w + 288)) || upload(r.stem_sc, sc) || upload(r.stem_sh, sh)) return DG_ECUDA;
  }
  int in_planes = 32, bi = 0;
  r.blocks.resize(16);
  for (int st = 0; st < 4; st++)
    for (int b = 0; b < RN_BLOCKS[st]; b++, bi++) {
      const int planes = RN_CH[st], stride = (b == 0 && st > 0) ? 2 : 1;
      const std::string pre = "resnet.layer" + std::to_string(st + 1) + "." + std::to_string(b) + ".";
      ResBlock& blk = r.blocks[bi];
      r.stage_of[bi] = st;
      if ((rc = resnet_conv_prepare(t, pre + "conv1", pre + "bn1", in_planes, planes, 3, stride, blk.c1)) ||
          (rc = resnet_conv_prepare(t, pre + "conv2", pre + "bn2", planes, planes, 3, 1, blk.c2)))
        return rc;
      blk.has_sc = stride != 1 || in_planes != planes;
      if (blk.has_sc && (rc = resnet_conv_prepare(t, pre + "shortcut.0", pre + "shortcut.1", in_planes, planes, 1, stride, blk.sc)))
        return rc;
      in_planes = planes;
    }
  // Linear(5120, D): pyannote's feature order is (channel, mel) -- "batch (dimension channel) frames" -- ours (mel, channel)
  const int64_t dn = t.numel("resnet.seg_1.bias");
  if (dn < 4 || dn % 4) {
    set_error("resnet.seg_1.bias missing or dimension not a multiple of 4");
    return DG_EWEIGHT;
  }
  h->D = (int)dn;
  const float* ew = t.get("resnet.seg_1.weight", dn * 5120);
  const float* eb = t.get("resnet.seg_1.bias", dn);
  if (!ew || !eb) return DG_EWEIGHT;
  std::vector<float> w_nk((size_t)dn * 5120);
  for (int o = 0; o < dn; o++)
    for (int half = 0; half < 2; half++)
      for (int hh = 0; hh < 10; hh++)
        for (int c = 0; c < 256; c++) w_nk[(size_t)o * 5120 + half * 2560 + hh * 256 + c] = ew[(size_t)o * 5120 + half * 2560 + c * 10 + hh];
  if (upload_split(h->ew, w_nk, (int)dn, ((int)dn + 255) / 256 * 256, 5120) ||
      upload(h->eb, std::vector<float>(eb, eb + dn)))
    return DG_ECUDA;
  h->pool_C = 2560;
  return 0;
}

// geometry of variant B for S samples: fbank frames and the four map sizes (time x mel)
struct ResGeom {
  int T0, W[4], H[4];
};
static int resnet_geom(int S, ResGeom& g) {
  if (S < 800 || S % 160) {
    set_error("WeSpeaker embedding: chunk length must be a multiple of 160 samples (>= 800)");
    return DG_EINVAL;
  }
  g.T0 = S / 160 - 2;                          // 1 + (S - 400) / 160, snip_edges
  g.W[0] = g.T0;
  g.H[0] = 80;
  for (int s = 1; s < 4; s++) {
    g.W[s] = (g.W[s - 1] - 1) / 2 + 1;
    g.H[s] = (g.H[s - 1] - 1) / 2 + 1;
  }
  return 0;
}

static int resnet_conv(const ResConv& c, const void* in_hi, const void* in_lo, int U, int Wp, int Hp, int Wop, int Hop,
                       void* out_hi, void* out_lo, float* out_f32, const void* res_hi, const void* res_lo, int relu,
                       const char* tag, cudaStream_t st) {
  int taps[9];
  if (c.ksize == 1) taps[0] = 0;
  else if (c.KW == 3)
    for (int dw = 0; dw < 3; dw++) taps[dw] = (dw - 1) * Hp - 1;           // three dh taps folded into one K slab
  else
    for (int dw = 0; dw < 3; dw++)
      for (int dh = 0; dh < 3; dh++) taps[dw * 3 + dh] = (dw - 1) * Hp + (dh - 1);
  TcGemm t{};
  const long long rows = (long long)U * Wp * Hp;
  t.A_hi = in_hi; t.A_lo = in_lo; t.lda = c.lda; t.Cin = c.cin_gemm; t.KW = c.KW; t.dil = 1; t.Mtot = rows; t.M = rows;
  t.N = c.cout; t.bn_scale = c.sc.as<float>(); t.bn_shift = c.sh.as<float>();
  t.out_hi = out_hi; t.out_lo = out_lo; t.out_f32 = out_f32; t.ldc = c.cout; t.epi = 3; t.tag = tag;
  t.tap_off = taps; t.Wp = Wp; t.Hp = Hp; t.Wop = Wop; t.Hop = Hop; t.stride2 = c.stride == 2; t.relu = relu;
  t.res_hi = res_hi; t.res_lo = res_lo;
  const int rc = set_weights(t, c.w);
  return rc ? rc : launch_gemm_tc(t, st);
}

// waveform [U,S] -> float32 final map [U][W3 + 2][H3 + 2][256] (h->pool_x descriptor), frames W3
static int resnet_trunk(dg_emb* h, const float* wav, int U, int S, cudaStream_t st, int* T_out) {
  int rc;
  ResNet& r = *h->rn;
  ResGeom g;
  if ((rc = resnet_geom(S, g))) return rc;
  const int rpi = S / 160;                                      // spectrum rows per item (the last two are not frames)
  const long long n = (long long)U * S;
  if (r.wav_hi.ensure(((size_t)n + 1024) * 2) || r.wav_lo.ensure(((size_t)n + 1024) * 2) ||
      r.spec.ensure(((size_t)U * rpi + 128) * 640 * 4) || r.logmel.ensure((size_t)U * g.T0 * 80 * 4) ||
      r.mean.ensure((size_t)U * 80 * 4) || r.inv_s.ensure((size_t)U * 4) ||
      r.level.ensure((size_t)U * (S / 80) * 4))
    return DG_ECUDA;
  for (int s = 0; s < 4; s++) {
    const size_t rows = (size_t)U * (g.W[s] + 2) * (g.H[s] + 2) + 256;      // + tail: overlapping-row reads of the last rows
    for (int b = 0; b < 3; b++)
      for (int p = 0; p < 2; p++)
        if (r.act[s][b][p].ensure(rows * RN_CH[s] * 2)) return DG_ECUDA;    // zero-initialised: the padding ring stays zero
  }
  if (r.fin.ensure(((size_t)U * (g.W[3] + 2) * (g.H[3] + 2) + 64) * 256 * 4)) return DG_ECUDA;
  if (r.last_S != S) {
    if (r.last_S)
      for (int s = 0; s < 4; s++)
        for (int b = 0; b < 3; b++)
          for (int p = 0; p < 2; p++) DG_CUDA(cudaMemsetAsync(r.act[s][b][p].p, 0, r.act[s][b][p].bytes, st));
    r.last_S = S;
  }
  // ---- kaldi fbank: planes of s (x * 2^15 - p), [rows, 448] x [448, 640] on the tensor cores, power -> mel -> log, time mean
  if ((rc = launch_fb_planes(wav, U, S, r.wav_hi.p, r.wav_lo.p, r.inv_s.as<float>(), r.level.as<float>(), st))) return rc;
  {
    TcGemm t{};
    t.A_hi = r.wav_hi.p; t.A_lo = r.wav_lo.p; t.lda = 160; t.Cin = 448; t.KW = 1; t.dil = 1;
    t.Mtot = (long long)U * rpi; t.M = (long long)U * rpi;
    t.N = 640; t.out_f32 = r.spec.as<float>(); t.ldc = 640; t.epi = 0; t.tag = "fbank_dft";
    if ((rc = set_weights(t, r.fb)) || (rc = launch_gemm_tc(t, st))) return rc;
  }
  if ((rc = launch_fb_mel(r.spec.as<float>(), 640, rpi, g.T0, U, r.inv_s.as<float>(), r.level.as<float>(), r.banks.as<float>(),
                          r.k_lo.as<int>(), r.k_hi.as<int>(), r.logmel.as<float>(), st)) ||
      (rc = launch_fb_mean(r.logmel.as<float>(), U, g.T0, r.mean.as<float>(), st)) ||
      (rc = launch_rn_stem(r.logmel.as<float>(), r.mean.as<float>(), U, g.T0, r.stem_w.as<float>(), r.stem_sc.as<float>(),
                           r.stem_sh.as<float>(), r.act[0][0][0].p, r.act[0][0][1].p, st)))
    return rc;
  // ---- 16 BasicBlocks: y = relu(bn1(conv1(x))); out = relu(bn2(conv2(y)) + shortcut(x))
  int cur = 0;                      // buffer (0 / 2) of the current stage that holds x
  int prev_stage = 0;
  static const char* kTags[4] = {"resnet_l1", "resnet_l2", "resnet_l3", "resnet_l4"};
  r.dbg_stage = 0;
  r.dbg_buf = 0;
  for (size_t bi = 0; bi < r.blocks.size() && (int)bi <= r.stop_after; bi++) {
    const ResBlock& blk = r.blocks[bi];
    const int s = r.stage_of[bi];
    const int Wp = g.W[s] + 2, Hp = g.H[s] + 2;
    DevBuf* x = r.act[prev_stage][cur];
    const int xWp = g.W[prev_stage] + 2, xHp = g.H[prev_stage] + 2;
    if (s != prev_stage) cur = 0;   // first block of a stage: x comes from the previous stage, the output goes to buffer 0
    DevBuf* y = r.act[s][1];
    DevBuf* out = s != prev_stage ? r.act[s][0] : r.act[s][cur ^ 2];
    const void *res_hi = x[0].p, *res_lo = x[1].p;
    if (blk.has_sc) {               // BatchNorm(Conv1x1 stride 2 (x)) into buffer 2 of this stage
      DevBuf* z = r.act[s][2];
      if ((rc = resnet_conv(blk.sc, x[0].p, x[1].p, U, xWp, xHp, Wp, Hp, z[0].p, z[1].p, nullptr, nullptr, nullptr, 0, kTags[s], st)))
        return rc;
      res_hi = z[0].p;
      res_lo = z[1].p;
    }
    if ((rc = resnet_conv(blk.c1, x[0].p, x[1].p, U, xWp, xHp, Wp, Hp, y[0].p, y[1].p, nullptr, nullptr, nullptr, 1, kTags[s], st)))
      return rc;
    const bool last = bi + 1 == r.blocks.size();
    if ((rc = resnet_conv(blk.c2, y[0].p, y[1].p, U, Wp, Hp, Wp, Hp, last ? nullptr : out[0].p, last ? nullptr : out[1].p,
                          last ? r.fin.as<float>() : nullptr, res_hi, res_lo, 1, kTags[s], st)))
      return rc;
    if (s == prev_stage) cur ^= 2;
    prev_stage = s;
    r.dbg_stage = s;
    r.dbg_buf = cur;
  }
  const int Wp3 = g.W[3] + 2, Hp3 = g.H[3] + 2;
  h->pool_x = r.fin.as<float>() + ((size_t)1 * Hp3 + 1) * 256;       // position (w = 1, h = 1) of item 0
  h->pool_item_pitch = (long long)Wp3 * Hp3 * 256;
  h->pool_row_pitch = Hp3 * 256;
  h->pool_C = g.H[3] * 256;
  *T_out = g.W[3];
  return 0;
}

// test hook: runs the variant-B trunk up to a given point and returns the intermediate map as float32 on the host.
// stop_after = -2: log-mel features [U][T0][80] (before mean normalisation), -1: stem output, k >= 0: output of BasicBlock k
// (dims = {U, W, H, C}, un-padded, layout [item][w = time][h = mel][channel]); 15 = the final map.
extern "C" int dg_emb_debug_trunk(dg_emb* h, const float* wav_dev, int U, int S, int stop_after, float* out_host, int64_t cap,
                                  int* dims) {
  if (!h || h->variant != 1 || !wav_dev || !out_host || !dims || U < 1) {
    set_error("dg_emb_debug_trunk: needs a WeSpeaker (variant B) handle");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  ResNet& r = *h->rn;
  ResGeom g;
  int rc, T = 0;
  if ((rc = resnet_geom(S, g))) return rc;
  r.stop_after = stop_after < -1 ? -1 : stop_after;
  rc = resnet_trunk(h, wav_dev, U, S, nullptr, &T);
  r.stop_after = 99;
  if (rc) return rc;
  DG_CUDA(cudaDeviceSynchronize());
  if (stop_after == -2) {
    dims[0] = U; dims[1] = g.T0; dims[2] = 80; dims[3] = 1;
    const int64_t n = (int64_t)U * g.T0 * 80;
    if (n > cap) return DG_EINVAL;
    DG_CUDA(cudaMemcpy(out_host, r.logmel.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return DG_OK;
  }
  const int s = r.dbg_stage, W = g.W[s], H = g.H[s], C = RN_CH[s], Wp = W + 2, Hp = H + 2;
  dims[0] = U; dims[1] = W; dims[2] = H; dims[3] = C;
  const int64_t n = (int64_t)U * W * H * C;
  if (n > cap) {
    set_error("dg_emb_debug_trunk: buffer too small");
    return DG_EINVAL;
  }
  const size_t rows = (size_t)U * Wp * Hp;
  std::vector<float> full(rows * C);
  if (stop_after >= 15) {
    DG_CUDA(cudaMemcpy(full.data(), r.fin.p, rows * C * 4, cudaMemcpyDeviceToHost));
  } else {
    std::vector<uint16_t> hi(rows * C), lo(rows * C);
    DG_CUDA(cudaMemcpy(hi.data(), r.act[s][r.dbg_buf][0].p, rows * C * 2, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(lo.data(), r.act[s][r.dbg_buf][1].p, rows * C * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < rows * C; i++) full[i] = host_h16_to_f32(hi[i]) + host_h16_to_f32(lo[i]);
  }
  for (int u = 0; u < U; u++)
    for (int w = 0; w < W; w++)
      for (int hh = 0; hh < H; hh++)
        memcpy(out_host + (((size_t)u * W + w) * H + hh) * C, &full[(((size_t)u * Wp + w + 1) * Hp + hh + 1) * C], (size_t)C * 4);
  return DG_OK;
}

extern "C" int dg_selftest_fbank_tables_host(float* frame_operator, float* mel_banks) {
  if (!frame_operator || !mel_banks) {
    set_error("dg_selftest_fbank_tables_host: null argument");
    return DG_EINVAL;
  }
  std::vector<float> op, banks;
  std::vector<int> lo, hi;
  fbank_frame_operator(op);
  fbank_mel_banks(banks, lo, hi);
  memcpy(frame_operator, op.data(), op.size() * sizeof(float));
  memcpy(mel_banks, banks.data(), banks.size() * sizeof(float));
  return DG_OK;
}

extern "C" int dg_emb_create(const dg_tensor* tensors, int n, int pool_mode, int device, dg_emb** out) {
  if (!tensors || !out || (pool_mode != 31 && pool_mode != 21)) {
    set_error("dg_emb_create: bad arguments (pool_mode must be 31 or 21)");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_emb> h(new dg_emb());
  h->device = device;
  h->pool_mode = pool_mode;
  Tensors t(tensors, n);
  int rc = emb_prepare(h.get(), t);
  if (rc) return rc;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_emb_dims(const dg_emb* h, int num_samples, int* frames, int* dimension) {
  if (!h || num_samples < 3000) {
    set_error("dg_emb_dims: bad arguments");
    return DG_EINVAL;
  }
  if (h->variant == 1) {
    ResGeom rg;
    int rc = resnet_geom(num_samples, rg);
    if (rc) return rc;
    if (frames) *frames = rg.W[3];
    if (dimension) *dimension = h->D;
    return DG_OK;
  }
  Geom g = make_geom(num_samples);
  if (frames) *frames = g.T2 - 14;
  if (dimension) *dimension = h->D;
  return DG_OK;
}

// F.interpolate index tables, computed in float32 exactly like ATen's upsample kernels
static int build_tables(dg_emb* h, int F, int T, cudaStream_t st) {
  if (h->tab_F == F && h->tab_T == T) return 0;
  std::vector<int> i0(T), i1(T);
  std::vector<float> l1(T);
  const float scale = (float)F / (float)T;
  for (int t = 0; t < T; t++) {
    if (F == T) {
      i0[t] = i1[t] = t;
      l1[t] = 0.f;
    } else if (h->pool_mode == 31) {   // mode="nearest": min(floor(dst * scale), F - 1)
      int s = (int)floorf((float)t * scale);
      if (s > F - 1) s = F - 1;
      i0[t] = i1[t] = s;
      l1[t] = 0.f;
    } else {                           // mode="linear", align_corners=False
      float src = scale * ((float)t + 0.5f) - 0.5f;
      if (src < 0.f) src = 0.f;
      int a = (int)src;
      if (a > F - 1) a = F - 1;
      i0[t] = a;
      i1[t] = a + (a < F - 1 ? 1 : 0);
      l1[t] = src - (float)a;
    }
  }
  if (h->idx0.ensure(T * 4) || h->idx1.ensure(T * 4) || h->lam1.ensure(T * 4)) return DG_ECUDA;
  DG_CUDA(cudaStreamSynchronize(st));
  DG_CUDA(cudaMemcpy(h->idx0.p, i0.data(), T * 4, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->idx1.p, i1.data(), T * 4, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->lam1.p, l1.data(), T * 4, cudaMemcpyHostToDevice));
  h->tab_F = F;
  h->tab_T = T;
  return 0;
}

// waveform [U,S] -> t5 [U*S2, 1500]; returns the number of valid frames.
// `defer_last`: stop before TDNN5 (its operand planes are left in h->t4h / t4l) -- the caller runs it fused with the pooling.
// `prep`: waveform statistics + planes the caller computed (or null)
int emb_trunk(dg_emb* h, const float* wav, int U, const Geom& g, cudaStream_t st, int* T_out, bool defer_last,
              const SincPrep* prep, int stop_after) {
  int rc;
  if (h->variant == 1) return resnet_trunk(h, wav, U, g.S, st, T_out);
  if ((rc = run_sincnet(h->sw, h->work, wav, U, g, st, prep))) return rc;
  const size_t rows = (size_t)U * g.S2 + 64;
  if (h->t5.ensure(rows * 1500 * 4)) return DG_ECUDA;
  h->pool_x = h->t5.as<float>();
  h->pool_item_pitch = (long long)g.S2 * 1500;
  h->pool_row_pitch = 1500;
  h->pool_C = 1500;
  const long long M = (long long)U * g.S2;
  if (h->xh.ensure(rows * 64 * 2) || h->xl.ensure(rows * 64 * 2) || h->aH.ensure(rows * 512 * 2) ||
      h->aL.ensure(rows * 512 * 2) || h->bH.ensure(rows * 512 * 2) || h->bL.ensure(rows * 512 * 2))
    return DG_ECUDA;
  if ((rc = launch_split_ex(h->work.out, M, 64, 64, 64, h->work.out_pool, g.S2, h->work.sc2.as<float>(),
                            h->work.sh2.as<float>(), h->xh.p, h->xl.p, st)))
    return rc;
  const void *ih = h->xh.p, *il = h->xl.p;
  int cin = 64, T = g.T2;
  void* oh[2] = {h->aH.p, h->bH.p};
  void* ol[2] = {h->aL.p, h->bL.p};
  static const char* kTags[5] = {"tdnn1", "tdnn2", "tdnn3", "tdnn4", "tdnn5"};
  for (int L = 0; L < 5 && stop_after >= 0; L++) {
    if (L == 4 && defer_last) {
      h->t4h = ih;
      h->t4l = il;
      T -= (TD_K[L] - 1) * TD_DIL[L];
      break;
    }
    TcGemm t{};
    t.A_hi = ih; t.A_lo = il; t.lda = cin; t.Cin = cin; t.KW = TD_K[L]; t.dil = TD_DIL[L]; t.Mtot = M; t.M = M;
    t.N = TD_OUT[L]; t.bias = h->tb[L].as<float>(); t.bn_scale = h->bns[L].as<float>(); t.bn_shift = h->bnh[L].as<float>();
    t.tag = kTags[L];
    if (L == 4) {
      t.out_f32 = h->t5.as<float>(); t.ldc = 1500; t.epi = 2;
    } else {
      t.out_hi = oh[L & 1]; t.out_lo = ol[L & 1]; t.ldc = 512; t.epi = 1;
    }
    if ((rc = set_weights(t, h->tw[L])) || (rc = launch_gemm_tc(t, st))) return rc;
    ih = oh[L & 1]; il = ol[L & 1];
    cin = TD_OUT[L];
    T -= (TD_K[L] - 1) * TD_DIL[L];
    if (L == stop_after) break;
  }
  *T_out = T;
  return 0;
}

// TDNN5 (Conv1d(512, 1500, 1) -> LeakyReLU -> BatchNorm) fused with the K weighted statistics poolings over the row weights
// `row_w` and weight sums `vsum` of launch_pool_weights: the [rows, 1500] map (455 MB at B = 256) is never written; the
// epilogue leaves per-tile partial sums, pool_finalize turns them into mean / std.
static int emb_tdnn5_pool_rows(dg_emb* h, int U, const Geom& g, const float* row_w, const float* vsum, int K, int T, float eps,
                               cudaStream_t st) {
  int rc;
  const long long M = (long long)U * g.S2;
  const int m_tiles = (int)((M + 127) / 128);
  if (h->pool_part.ensure((size_t)m_tiles * 2 * TC_POOL_SLOTS * 1500 * 4) || h->pooled.ensure((size_t)U * K * 3000 * 4)) return DG_ECUDA;
  TcGemm t{};
  t.A_hi = h->t4h; t.A_lo = h->t4l; t.lda = 512; t.Cin = 512; t.KW = 1; t.dil = 1; t.Mtot = M; t.M = M;
  t.N = 1500; t.bias = h->tb[4].as<float>(); t.bn_scale = h->bns[4].as<float>(); t.bn_shift = h->bnh[4].as<float>();
  t.ldc = 1500; t.epi = 4; t.tag = "tdnn5";
  t.pool_w = row_w; t.pool_part = h->pool_part.as<float>(); t.pool_item_rows = g.S2; t.pool_K = K; t.pool_T = T;
  if ((rc = set_weights(t, h->tw[4])) || (rc = launch_gemm_tc(t, st))) return rc;
  h->pool_C = 1500;
  return launch_pool_finalize(h->pool_part.as<float>(), row_w, vsum, h->bnh[4].as<float>(), U, K, 1500, g.S2, T, eps,
                              h->pooled.as<float>(), st);
}

static int emb_tdnn5_pool(dg_emb* h, int U, const Geom& g, const float* weights, int F, int K, int T, float eps,
                          cudaStream_t st) {
  int rc;
  const long long M = (long long)U * g.S2;
  if (h->pool_rw.ensure(((size_t)M + 128) * 16) || h->pool_vs.ensure((size_t)U * K * 8)) return DG_ECUDA;
  if ((rc = launch_pool_weights(weights, U, F, K, g.S2, T, h->idx0.as<int>(), h->idx1.as<int>(), h->lam1.as<float>(), eps,
                                h->pool_rw.as<float>(), h->pool_vs.as<float>(), st)))
    return rc;
  return emb_tdnn5_pool_rows(h, U, g, h->pool_rw.as<float>(), h->pool_vs.as<float>(), K, T, eps, st);
}

static int emb_project(dg_emb* h, int rows, int normalize, float norm, float* out, cudaStream_t st) {
  int rc;
  const int nfeat = 2 * h->pool_C, kpad = (nfeat + 63) / 64 * 64;     // 3000 -> 3008, 5120 -> 5120
  if (h->ph.ensure(((size_t)rows + 128) * kpad * 2) || h->pl.ensure(((size_t)rows + 128) * kpad * 2)) return DG_ECUDA;
  if ((rc = launch_split_ex(h->pooled.as<float>(), rows, nfeat, nfeat, kpad, 0, 1, nullptr, nullptr, h->ph.p, h->pl.p, st)))
    return rc;
  float* dst = out;
  if (normalize) {
    if (h->eraw.ensure((size_t)rows * h->D * 4)) return DG_ECUDA;
    dst = h->eraw.as<float>();
  }
  TcGemm t{};
  t.A_hi = h->ph.p; t.A_lo = h->pl.p; t.lda = kpad; t.Cin = kpad; t.KW = 1; t.dil = 1; t.Mtot = rows; t.M = rows;
  t.N = h->D; t.bias = h->eb.as<float>(); t.out_f32 = dst; t.ldc = h->D; t.epi = 0; t.tag = "emb_linear";
  if ((rc = set_weights(t, h->ew)) || (rc = launch_gemm_tc(t, st))) return rc;
  return normalize ? launch_l2norm(dst, rows, h->D, norm, out, st) : 0;
}

// epsilon of the weighted statistics pooling: 1e-8 for pyannote's StatsPool with weights, none without them
static float pool_eps(const dg_emb* h, const float* weights) { return weights && h->pool_mode == 31 ? 1e-8f : 0.f; }

// the pooling can run fused with TDNN5 (emb_tdnn5_pool) for pooling weights of this many speakers at this chunk size
bool pool_fusable(const dg_emb* h, int K, const Geom& g) { return h->variant == 0 && K <= 4 && g.S2 >= 128; }


// Everything after the embedding trunk: interpolation tables, the K weighted statistics poolings of each item -- fused with
// TDNN5 when `fuse` (the trunk was run with defer_last) -- and the projection, into out [B*K, D].  `sm_cap` caps the grids of
// the fused part (the un-fused pooling and its projection are not capped).
int emb_tail(dg_emb* h, int B, const Geom& g, const float* weights, int F, int K, int T, bool fuse, int normalize,
             float norm, float* out, cudaStream_t st, int sm_cap) {
  int rc;
  if (weights && (rc = build_tables(h, F, T, st))) return rc;
  const float eps = pool_eps(h, weights);
  if (fuse) {
    SmLimit cap(sm_cap);
    if ((rc = emb_tdnn5_pool(h, B, g, weights, F, K, T, eps, st))) return rc;
    return emb_project(h, B * K, normalize, norm, out, st);
  }
  if (h->pooled.ensure((size_t)B * K * 2 * h->pool_C * 4)) return DG_ECUDA;
  if ((rc = launch_stats_pool(h->pool_x, B, g.S2, T, h->pool_C, weights, F, K, h->idx0.as<int>(), h->idx1.as<int>(),
                              h->lam1.as<float>(), eps, h->pooled.as<float>(), st, h->pool_item_pitch, h->pool_row_pitch)))
    return rc;
  return emb_project(h, B * K, normalize, norm, out, st);
}

// emb_tail for G OSP sets over one trunk pass: weights [G][B][F][K], set g's embeddings [B*K, D] at out + g out_stride.  The
// fused form computes the row weights of all sets in one launch and then runs TDNN5 + pooling, the finaliser and the projection
// once per set over the kept TDNN5 operand planes; the un-fused form runs emb_tail per set over the kept trunk map.  Either way
// set g's embeddings are the bits emb_tail gives for weights g.
int emb_tail_sets(dg_emb* h, int B, const Geom& g, const float* weights, int G, int F, int K, int T, bool fuse, float* out,
                  int64_t out_stride, cudaStream_t st, int sm_cap) {
  int rc;
  const size_t wstride = (size_t)B * F * K;
  if (!fuse) {
    for (int s = 0; s < G; s++)
      if ((rc = emb_tail(h, B, g, weights + s * wstride, F, K, T, false, 1, 1.f, out + s * out_stride, st))) return rc;
    return 0;
  }
  if ((rc = build_tables(h, F, T, st))) return rc;
  const float eps = pool_eps(h, weights);
  const long long M = (long long)B * g.S2, rw_stride = (M + 128) * 4;
  if (h->pool_rw.ensure((size_t)G * rw_stride * 4) || h->pool_vs.ensure((size_t)G * B * K * 8)) return DG_ECUDA;
  SmLimit cap(sm_cap);
  if ((rc = launch_pool_weights_sets(weights, B, G, F, K, g.S2, T, h->idx0.as<int>(), h->idx1.as<int>(), h->lam1.as<float>(), eps,
                                     h->pool_rw.as<float>(), rw_stride, h->pool_vs.as<float>(), st)))
    return rc;
  for (int s = 0; s < G; s++)
    if ((rc = emb_tdnn5_pool_rows(h, B, g, h->pool_rw.as<float>() + s * rw_stride, h->pool_vs.as<float>() + (size_t)s * B * K * 2,
                                  K, T, eps, st)) ||
        (rc = emb_project(h, B * K, 1, 1.f, out + s * out_stride, st)))
      return rc;
  return 0;
}

extern "C" int dg_emb_forward(dg_emb* h, const float* wav, const float* weights, int B, int S, int F, int K,
                              int normalize, float norm, float* out, void* stream) {
  if (!h || !wav || !out || B < 1 || S < 3000 || K < 1 || (!weights && K != 1) || (weights && F < 1)) {
    set_error("dg_emb_forward: bad arguments");
    return DG_EINVAL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  DG_CUDA(cudaSetDevice(h->device));
  const Geom g = make_geom(S);
  int rc, T = 0;
  LaneUse use(h->guard, stream ? stream : (void*)h, st);
  if ((rc = use.rc)) return rc;
  const bool fuse = weights && pool_fusable(h, K, g);
  if ((rc = emb_trunk(h, wav, B, g, st, &T, fuse, nullptr))) return rc;
  return emb_tail(h, B, g, weights, F, K, T, fuse, normalize, norm, out, st);
}

// test hook: the production front end, emb_trunk and emb_tail with a host-side stop point, and one intermediate map copied to
// the host.  Stages 9 / 11 take the fused TDNN5 + pooling (refused where pool_fusable says no), 10 / 12 the un-fused pooling.
extern "C" int dg_emb_debug_stage(dg_emb* h, const float* wav_dev, const float* weights_dev, int B, int S, int F, int K, int hop,
                                  int stage, float* out_host, int64_t cap, int* dims) {
  if (!h || !wav_dev || !out_host || !dims || B < 1 || S < 3000 || hop < 0 || stage < 0 || stage > 12 ||
      (stage >= 9 && (!weights_dev || F < 1 || K < 1)) || h->variant != 0) {
    set_error("dg_emb_debug_stage: bad arguments (need an XVectorSincNet handle, B >= 1, S >= 3000, stage 0..12, weights from stage 9)");
    return DG_EINVAL;
  }
  const Geom g = make_geom(S);
  const bool fuse = stage == 9 || stage == 11;
  if (fuse && !pool_fusable(h, K, g)) {
    set_error("dg_emb_debug_stage: the fused pooling does not run at this K and chunk length");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  const char* who = "dg_emb_debug_stage";
  cudaStream_t st = nullptr;
  SincPrep shared;
  const SincPrep* prep = nullptr;
  DevBuf out;
  int rc, T = 0;
  if (stage >= 9 && out.ensure((size_t)B * K * h->D * 4)) return DG_ECUDA;
  {
    LaneUse use(h->guard, h, st);
    if ((rc = use.rc)) return rc;
    if (hop > 0) {
      if ((rc = run_sinc_prep(shared, wav_dev, B, g, st, hop, false))) return rc;
      prep = &shared;
    }
    if ((rc = emb_trunk(h, wav_dev, B, g, st, &T, fuse, prep, stage <= 3 ? -1 : stage <= 7 ? stage - 4 : 99))) return rc;
    if (stage >= 9 && (rc = emb_tail(h, B, g, weights_dev, F, K, T, fuse, 0, 1.f, out.as<float>(), st))) return rc;
  }
  DG_CUDA(cudaDeviceSynchronize());
  if ((rc = debug_front_paths(prep, g, &dims[3]))) return rc;
  if (fuse) dims[3] |= DG_DBG_STATS_POOL_FUSED;
  if (stage <= 3) return debug_copy_front(who, stage, h->work, prep, h->xh.p, h->xl.p, B, g, out_host, cap, dims);
  if (stage <= 7) {
    const int L = stage - 4;
    return debug_copy_map(who, L & 1 ? h->bH.p : h->aH.p, L & 1 ? h->bL.p : h->aL.p, B, g.S2, 512, T, 512, out_host, cap, dims);
  }
  if (stage == 8) return debug_copy_map(who, h->t5.p, nullptr, B, g.S2, 1500, T, 1500, out_host, cap, dims);
  if (stage <= 10) return debug_copy_map(who, h->pooled.p, nullptr, B * K, 1, 3000, 1, 3000, out_host, cap, dims);
  return debug_copy_map(who, out.p, nullptr, B * K, 1, h->D, 1, h->D, out_host, cap, dims);
}

extern "C" int dg_emb_forward_rows(dg_emb* h, const float* wav, const float* weights, int N, int S, int F, float* out,
                                   void* stream) {
  if (!h || !wav || !out || N < 1 || S < 3000 || (weights && F < 1)) {
    set_error("dg_emb_forward_rows: bad arguments");
    return DG_EINVAL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  DG_CUDA(cudaSetDevice(h->device));
  const Geom g = make_geom(S);
  int rc, T = 0;
  LaneUse use(h->guard, stream ? stream : (void*)h, st);
  if ((rc = use.rc)) return rc;
  // consecutive identical rows (the reference repeats each waveform once per local speaker,
  // src/diart/blocks/embedding.py:57-59) share one trunk pass
  if (h->flags.ensure((size_t)N * 4)) return DG_ECUDA;
  if ((rc = launch_row_equal_flags(wav, N, S, h->flags.as<int>(), st))) return rc;
  std::vector<int> flags(N);
  DG_CUDA(cudaMemcpyAsync(flags.data(), h->flags.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaStreamSynchronize(st));
  std::vector<int> uniq, gi, gq0, gnq;
  for (int n = 0; n < N; n++) {
    if (!flags[n]) uniq.push_back(n);
    const int item = (int)uniq.size() - 1;
    if (!flags[n] || gnq.back() == 4) {
      gi.push_back(item);
      gq0.push_back(n);
      gnq.push_back(1);
    } else {
      gnq.back()++;
    }
  }
  const int U = (int)uniq.size(), G = (int)gi.size();
  const float* trunk_in = wav;
  if (U != N) {
    if (h->uniq.ensure((size_t)U * 4) || h->gathered.ensure((size_t)U * S * 4)) return DG_ECUDA;
    DG_CUDA(cudaMemcpyAsync(h->uniq.p, uniq.data(), (size_t)U * 4, cudaMemcpyHostToDevice, st));
    if ((rc = launch_gather_rows(wav, h->uniq.as<int>(), U, S, h->gathered.as<float>(), st))) return rc;
    trunk_in = h->gathered.as<float>();
  }
  if (h->grp.ensure((size_t)3 * G * 4)) return DG_ECUDA;
  std::vector<int> packed(3 * G);
  memcpy(packed.data(), gi.data(), G * 4);
  memcpy(packed.data() + G, gq0.data(), G * 4);
  memcpy(packed.data() + 2 * G, gnq.data(), G * 4);
  DG_CUDA(cudaMemcpyAsync(h->grp.p, packed.data(), (size_t)3 * G * 4, cudaMemcpyHostToDevice, st));
  if ((rc = emb_trunk(h, trunk_in, U, g, st, &T, false, nullptr))) return rc;
  if (weights && (rc = build_tables(h, F, T, st))) return rc;
  if (h->pooled.ensure((size_t)N * 2 * h->pool_C * 4)) return DG_ECUDA;
  const int* gp = h->grp.as<int>();
  if ((rc = launch_stats_pool_ex(h->pool_x, g.S2, T, h->pool_C, weights, F, 1, 1, G, gp, gp + G, gp + 2 * G,
                                 h->idx0.as<int>(), h->idx1.as<int>(), h->lam1.as<float>(), pool_eps(h, weights),
                                 h->pooled.as<float>(), st, h->pool_item_pitch, h->pool_row_pitch)))
    return rc;
  rc = emb_project(h, N, 0, 1.f, out, st);
  DG_CUDA(cudaStreamSynchronize(st));   // host staging vectors above must outlive the async copies
  return rc;
}

extern "C" int dg_emb_destroy(dg_emb* h) {
  delete h;
  return DG_OK;
}

// =========================================================================== element-wise blocks
extern "C" int dg_osp(const float* seg, int B, int F, int K, float gamma, float beta, int normalize, float* out,
                      void* stream) {
  if (!seg || !out || B < 1 || F < 1 || K < 1) {
    set_error("dg_osp: bad arguments");
    return DG_EINVAL;
  }
  return launch_osp(seg, B, F, K, gamma, beta, normalize, out, (cudaStream_t)stream);
}

extern "C" int dg_normalize_embeddings(const float* emb, int rows, int D, float norm, float* out, void* stream) {
  if (!emb || !out || rows < 1 || D < 1) {
    set_error("dg_normalize_embeddings: bad arguments");
    return DG_EINVAL;
  }
  return launch_l2norm(emb, rows, D, norm, out, (cudaStream_t)stream);
}

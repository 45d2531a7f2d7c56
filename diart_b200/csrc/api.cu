// C ABI of libdiartb200.so (include/diart_b200.h): handles, weight preparation, workspaces and the
// launch sequences of the two networks, the clustering step and the fused pipeline step.
#include <math.h>
#include <cmath>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <deque>
#include <map>
#include <memory>
#include <sstream>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <numeric>
#include <atomic>
#include <chrono>
#include <thread>
#include <vector>

#include "../../include/diart_b200.h"
#include "dg_common.cuh"

namespace dg {

static thread_local std::string g_err;
std::atomic<long long> g_launches{0};
thread_local int g_sm_limit = 0;   // per host thread: distinct handles driven by distinct threads stay independent
void set_error(const std::string& msg) { g_err = msg; }

struct ProfRec {
  std::string name;
  cudaEvent_t a, b;
};
static bool g_prof = false;
static std::vector<ProfRec> g_recs;
// DG_TRACE_LAUNCHES=1: every scope prints "dg-trace <tag> <first launch ordinal> <one past the last>" on stderr, so that a
// profiler's launch list (tools/ncu_summary.py) can be labelled with the tags bench.py reports
static const bool g_trace = getenv("DG_TRACE_LAUNCHES") && getenv("DG_TRACE_LAUNCHES")[0] == '1';
ProfScope::ProfScope(const char* name_, cudaStream_t st_) : on(g_prof), st(st_), a(nullptr), b(nullptr), name(name_) {
  if (g_trace) first = g_launches.load();
  if (!on) return;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a, st);
}
ProfScope::~ProfScope() {
  if (g_trace) fprintf(stderr, "dg-trace %s %lld %lld\n", name, first, (long long)g_launches.load());
  if (!on) return;
  cudaEventRecord(b, st);
  g_recs.push_back({name, a, b});
}

int launch_stats_pool_ex(const float* x, int stride, int T, int C, const float* w, int F, int K, int layout,
                         int n_groups, const int* grp_item, const int* grp_q0, const int* grp_nq, const int* idx0,
                         const int* idx1, const float* lam1, float eps, float* pooled, cudaStream_t st,
                         long long item_pitch = 0, int row_pitch = 0);

// ------------------------------------------------------------------------------ small utilities
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  int ensure(size_t n) {
    if (n <= bytes) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    // (re)allocation is rare (first step at a given batch size).  The handles drive several non-blocking
    // streams, which do not order against the legacy stream this memset runs on: drain the device on both sides.
    DG_CUDA(cudaDeviceSynchronize());
    DG_CUDA(cudaMalloc(&p, n));
    DG_CUDA(cudaMemset(p, 0, n));
    DG_CUDA(cudaDeviceSynchronize());
    bytes = n;
    return 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

// An owned CUDA handle, freed by `Free`; movable, not copyable.  A handle struct that holds its streams, events and pinned
// memory this way frees everything it created, also when its creation fails halfway.
template <class H, cudaError_t (*Free)(H)>
struct Owned {
  H h = nullptr;
  Owned() = default;
  Owned(Owned&& o) noexcept : h(o.h) { o.h = nullptr; }
  Owned& operator=(Owned&& o) noexcept {
    std::swap(h, o.h);
    return *this;
  }
  ~Owned() {
    if (h) Free(h);
  }
  operator H() const { return h; }
};
struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
  int create(int priority = 0) {   // 0: the default priority
    DG_CUDA(cudaStreamCreateWithPriority(&h, cudaStreamNonBlocking, priority));
    return 0;
  }
};
struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
  int create() {
    DG_CUDA(cudaEventCreateWithFlags(&h, cudaEventDisableTiming));
    return 0;
  }
};
struct PinnedBuf : Owned<void*, cudaFreeHost> {
  size_t bytes = 0;
  int ensure(size_t n) {   // like DevBuf::ensure, without clearing
    if (n <= bytes) return 0;
    if (h) cudaFreeHost(h);
    h = nullptr;
    bytes = 0;
    DG_CUDA(cudaHostAlloc(&h, n, cudaHostAllocDefault));
    bytes = n;
    return 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(h); }
};

// A model handle owns ONE set of activation buffers per scratch lane.  A new user of a lane -- another pipeline built on the same
// handle, or a block-level call on another stream -- first waits, stream-ordered, for the previous user's last kernel; without it
// two users in flight would silently overwrite each other's activations.  (Host threads: a handle is single-threaded.)
struct UseGuard {
  Event e;                       // recorded at the end of the last use
  const void* owner = nullptr;   // who made it
};
// One use of a lane by `owner` on `st`: the constructor makes `st` wait for a previous user's end (`rc` = its result); end(), or
// the destructor on any other exit, records this use's end, so that the next user also waits for what an error left enqueued.
struct LaneUse {
  UseGuard& u;
  const void* owner;
  cudaStream_t st;
  int rc;
  bool open = true;
  LaneUse(UseGuard& u_, const void* owner_, cudaStream_t st_) : u(u_), owner(owner_), st(st_), rc(begin()) {}
  ~LaneUse() { end(); }
  int end() {
    if (!open) return 0;
    open = false;
    if (!u.e && u.e.create()) return DG_ECUDA;
    DG_CUDA(cudaEventRecord(u.e, st));
    u.owner = owner;
    return 0;
  }
  int begin() {
    if (u.e && u.owner != owner) DG_CUDA(cudaStreamWaitEvent(st, u.e, 0));
    return 0;
  }
};

struct Tensors {
  std::map<std::string, std::pair<const float*, int64_t>> m;
  Tensors(const dg_tensor* t, int n) {
    for (int i = 0; i < n; i++)
      if (t[i].name) m[t[i].name] = {t[i].data, t[i].numel};
  }
  const float* get(const std::string& name, int64_t numel) const {
    auto it = m.find(name);
    if (it == m.end()) {
      set_error("missing tensor '" + name + "' in state dict");
      return nullptr;
    }
    if (it->second.second != numel || !it->second.first) {
      set_error("tensor '" + name + "' has " + std::to_string(it->second.second) + " elements, expected " +
                std::to_string(numel));
      return nullptr;
    }
    return it->second.first;
  }
  int64_t numel(const std::string& name) const {
    auto it = m.find(name);
    return it == m.end() ? -1 : it->second.second;
  }
};

static int upload_u16(DevBuf& b, const std::vector<uint16_t>& h) {
  if (b.ensure(h.size() * 2)) return -2;
  DG_CUDA(cudaMemcpy(b.p, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  return 0;
}

// The B operand of a tensor-core GEMM: fp16 hi/lo planes [Npad][K] of float32 weights that were multiplied by `scale` (a power
// of two) before the split.  Npad, the row count the GEMM's tiles read, is decided here once, at upload.
struct WeightPlanes {
  DevBuf hi, lo;
  float scale = 1.f;
  int Npad = 0, K = 0;
};

// float32 [N][K] host weights -> zero-padded planes [Npad][K]
static int upload_split(WeightPlanes& w, const std::vector<float>& w_nk, int N, int Npad, int K) {
  std::vector<uint16_t> h((size_t)Npad * K), l((size_t)Npad * K);
  w.scale = weight_plane_scale(w_nk.data(), (size_t)N * K);
  w.Npad = Npad;
  w.K = K;
  split_weights_host(w_nk.data(), N, Npad, K, h.data(), l.data(), w.scale);
  return (upload_u16(w.hi, h) || upload_u16(w.lo, l)) ? DG_ECUDA : 0;
}

// points `t` at its weight planes; the launch's taps and channels (KW, Cin) must span exactly the planes' K
static int set_weights(TcGemm& t, const WeightPlanes& w) {
  if (t.KW * t.Cin != w.K) {
    set_error(std::string(t.tag ? t.tag : "gemm_tc") + ": the launch reads K = " + std::to_string(t.KW * t.Cin) +
              " but the weight planes have K = " + std::to_string(w.K));
    return DG_EINVAL;
  }
  t.W_hi = w.hi.p;
  t.W_lo = w.lo.p;
  t.w_scale = w.scale;
  t.Npad = w.Npad;
  return 0;
}

static int upload(DevBuf& b, const std::vector<float>& h) {
  if (b.ensure(h.size() * sizeof(float))) return -2;
  DG_CUDA(cudaMemcpy(b.p, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

// ------------------------------------------------------------------------------ SincNet front end
struct SincWeights {
  float wn_gamma = 1.f, wn_beta = 0.f;
  DevBuf g0, b0, bias1, g1, b1, bias2, g2, b2;
  WeightPlanes w1, w2;                 // conv weights [64][448] (taps folded into K: 5 x 80 + pad) and [64][5*64]
  DevBuf filt_planes;                  // sinc filter bank as fp16 planes [2][80][256] (hi, lo)
  DevBuf cf;                           // folded wav-norm affine: beta * sum_k h[f][k]
  DevBuf hsum;                         // sum_k h[f][k] (stream form of the sinc layer)
};

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

static int prep_sincnet(const Tensors& t, const std::string& pre, SincWeights& w) {
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
    // Conv1d(80, 60, 5) with its taps folded into K: the input planes are 80-channel rows (pitch 160 B), so the im2col row of
    // output row m is the 400 CONTIGUOUS values starting at row m -- read through an overlapping-row TMA view, K = 448
    const float* s1 = t.get(pre + "conv1d.1.weight", (int64_t)60 * 80 * 5);
    if (!s1) return DG_EWEIGHT;
    std::vector<float> w_nk((size_t)60 * 448, 0.f);
    for (int o = 0; o < 60; o++)
      for (int c = 0; c < 80; c++)
        for (int j = 0; j < 5; j++) w_nk[(size_t)o * 448 + j * 80 + c] = s1[((size_t)o * 80 + c) * 5 + j];
    if (upload_split(w.w1, w_nk, 60, 64, 448)) return DG_ECUDA;
  }
  if ((rc = conv_w_tc(pre + "conv1d.2.weight", 60, 60, 5, 64, w.w2))) return rc;
  return 0;
}

// waveform statistics and the standardised-waveform planes of a batch; both networks' SincNets read the same
// ones, so the fused pipeline computes them once per step
struct SincPrep {
  DevBuf wmean, wrstd, wh, wl;
  // stream form (needs a hop hint): planes of the raw stream and the device flag "this batch is a run of overlapping
  // windows"; `hop` > 0 means the stream-form launches were enqueued for this batch
  DevBuf swh, swl, flag, spart;
  int hop = 0;
  int ensure(int B, const Geom& g) {
    const size_t bytes = 4 * sinc_tc_plane_elems(B, g) * 2;
    return (wmean.ensure(B * 4) || wrstd.ensure(B * 4) || wh.ensure(bytes) || wl.ensure(bytes)) ? DG_ECUDA : 0;
  }
  int ensure_stream(int B, const Geom& g, int hop_) {
    const size_t bytes = 4 * sinc_stream_geom(B, g, hop_).plane * 2;
    return (swh.ensure(bytes) || swl.ensure(bytes) || flag.ensure(16)) ? DG_ECUDA : 0;
  }
};
struct SincWork {
  DevBuf p0, sc0, sh0, p1, sc1, sh1, p2, sc2, sh2;
  DevBuf a0h, a0l, c1, a1h, a1l, c2;   // fp16 planes of the conv inputs; un-pooled conv outputs of the un-fused path
  DevBuf craw, part;                   // stream form: raw convolution of the stream [P][80], statistics partials
  DevBuf part3;                        // per-tile InstanceNorm partial sums of the pooling GEMM epilogues (conv1, conv2)
  SincPrep own_prep;                   // statistics + waveform planes when no shared ones are supplied
  const float* out = nullptr;          // conv2 output that the next layer normalises on load ...
  int out_pool = 0;                    // ... 1: still un-pooled (rows = 3x), MaxPool1d(3) is applied on load
  int ensure(int B, const Geom& g) {
    const size_t tail = 64;  // spare rows so shifted windows of the last tile stay in bounds
    if (p0.ensure(((size_t)B * g.S0 + tail) * 80 * 4) || sc0.ensure((size_t)B * 80 * 4) || sh0.ensure((size_t)B * 80 * 4) ||
        p1.ensure(((size_t)B * g.S1 + tail) * 64 * 4) || sc1.ensure((size_t)B * 64 * 4) ||
        sh1.ensure((size_t)B * 64 * 4) || p2.ensure(((size_t)B * g.S2 + tail) * 64 * 4) ||
        sc2.ensure((size_t)B * 64 * 4) || sh2.ensure((size_t)B * 64 * 4) ||
        a0h.ensure(((size_t)B * g.S0 + tail) * 128 * 2) || a0l.ensure(((size_t)B * g.S0 + tail) * 128 * 2) ||
        c1.ensure(((size_t)B * g.S0 + tail) * 64 * 4) || a1h.ensure(((size_t)B * g.S1 + tail) * 64 * 2) ||
        a1l.ensure(((size_t)B * g.S1 + tail) * 64 * 2) || c2.ensure(((size_t)B * g.S1 + tail) * 64 * 4))
      return DG_ECUDA;
    return 0;
  }
};

static int run_sinc_prep(SincPrep& p, const float* wav, int B, const Geom& g, cudaStream_t st, int hop = 0,
                         bool overlap_known = false) {
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
  if (p.hop && (rc = launch_stream_prep(wav, B, g, hop, p.swh.p, p.swl.p, p.flag.as<int>(), st))) return rc;
  return launch_sinc_prep(wav, p.wmean.as<float>(), p.wrstd.as<float>(), B, g, p.wh.p, p.wl.p, st,
                          p.hop ? p.flag.as<int>() : nullptr);
}

// waveform [B,S] -> k.out (pre-norm conv2 output, pooled [B*S2,64] or un-pooled [B*S1,64]) + its
// InstanceNorm scale/shift (k.sc2, k.sh2)
static int run_sincnet(const SincWeights& w, SincWork& k, const float* wav, int B, const Geom& g, cudaStream_t st,
                       const SincPrep* shared = nullptr) {
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
  // never written, the statistics pass reads 2 x 2 x 64 floats per tile.  Needs a tile of 96..126 rows that divides the item at both
  // stages; otherwise the un-pooled float32 map -> instnorm_stats -> split with pooling on load
  const int tr0 = gemm_tc_pool3_tile_rows(g.S0), tr1 = gemm_tc_pool3_tile_rows(g.S1);
  if (tr0 && tr1) {
    if (k.part3.ensure((size_t)(M0 / tr0) * 2 * 2 * 64 * 4)) return DG_ECUDA;
    TcGemm t{};
    t.A_hi = k.a0h.p; t.A_lo = k.a0l.p; t.lda = 80; t.Cin = 448; t.KW = 1; t.dil = 1; t.Mtot = M0; t.M = M0;
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
  t.A_hi = k.a0h.p; t.A_lo = k.a0l.p; t.lda = 80; t.Cin = 448; t.KW = 1; t.dil = 1; t.Mtot = M0; t.M = M0;
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

}  // namespace dg

using namespace dg;

// ================================================================================== segmentation
struct dg_seg {
  int device = 0, K = 3;           // K = classifier outputs (local speakers; powerset classes for powerset models)
  int ps_speakers = 0;             // > 0: powerset model with this many local speakers (dg_seg_set_powerset)
  DevBuf ps_masks;                 // speaker bit set of every powerset class
  SincWeights sw;
  DevBuf bih[4];                   // input projection bias b_ih + b_hh [1024]
  WeightPlanes wih[4];             // input projections [1024][in_pad]
  WeightPlanes whh[4];             // W_hh [2][512][128] as lstm_tc_pack_whh lays it out (hi, lo, scale; no GEMM shape)
  DevBuf l1b, l2b, cw, cb;
  WeightPlanes l1, l2;             // head Linears [128][in]
  DevBuf ones128, zeros128;
  // activations: two independent sets ("lanes") so that the fused pipeline can run the segmentation chains of
  // two consecutive steps concurrently (the recurrence occupies only 32 SMs)
  struct Scratch {
    SincWork work;
    DevBuf gx, y2;
    DevBuf xh, xl;                 // fp16 hi/lo planes of the current in-projection input
    DevBuf y1h, y1l;               // fp16 planes of the first head Linear's output
  } scr[2];
  UseGuard guard[2];               // per scratch lane
};

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

extern "C" const char* dg_last_error(void) { return g_err.c_str(); }
extern "C" int dg_version(void) { return 100; }
extern "C" int64_t dg_launch_count(void) { return (int64_t)g_launches.load(); }

extern "C" int dg_profile_enable(int enable) {
  g_prof = enable != 0;
  return DG_OK;
}

// JSON {"name": {"count": n, "ms": total}, ...} of everything recorded since the last report.
// Synchronises the device.  Returns the number of bytes written (excluding the terminator).
extern "C" int dg_profile_report(char* buf, int cap) {
  cudaDeviceSynchronize();
  std::map<std::string, std::pair<int, double>> agg;
  for (auto& r : g_recs) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.a, r.b);
    auto& e = agg[r.name];
    e.first++;
    e.second += ms;
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  g_recs.clear();
  std::ostringstream os;
  os << "{";
  bool first = true;
  for (auto& kv : agg) {
    if (!first) os << ", ";
    first = false;
    os << "\"" << kv.first << "\": {\"count\": " << kv.second.first << ", \"ms\": " << kv.second.second << "}";
  }
  os << "}";
  const std::string s = os.str();
  if (!buf || cap <= (int)s.size()) {
    set_error("dg_profile_report: buffer too small");
    return DG_EINVAL;
  }
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int)s.size();
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

// the forward on scratch lane `lane`, without the use bracket; `prep`: waveform statistics + planes the caller computed (or null)
static int seg_forward_lane(dg_seg* h, int lane, const SincPrep* prep, const float* wav, int B, int S, float* seg,
                            cudaStream_t st) {
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
  for (int L = 0; L < 4; L++) {
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

extern "C" int dg_seg_destroy(dg_seg* h) {
  delete h;
  return DG_OK;
}

// ===================================================================================== embedding
struct dg_emb {
  int device = 0, pool_mode = 31, D = 512;
  SincWeights sw;
  DevBuf tb[5], bns[5], bnh[5];
  WeightPlanes tw[5];                    // TDNN weights [Npad][K]
  WeightPlanes ew;                       // Linear(3000, D) weights [Dpad][3008] (WeSpeaker: Linear(5120, D))
  DevBuf ph, pl;                         // pooled statistics planes
  DevBuf xh, xl, aH, aL, bH, bL;         // fp16 hi/lo activation planes
  DevBuf eb;
  SincWork work;
  UseGuard guard;
  DevBuf t5, pooled, eraw;
  DevBuf idx0, idx1, lam1;
  int tab_F = -1, tab_T = -1;
  DevBuf flags, uniq, grp, gathered;   // compatibility path
  // what the pooling reads after a trunk pass: x(item, t, c) = pool_x[item * pool_item_pitch + t * pool_row_pitch + c], c < pool_C
  const float* pool_x = nullptr;
  long long pool_item_pitch = 0;
  int pool_row_pitch = 0, pool_C = 1500;
  const void *t4h = nullptr, *t4l = nullptr;   // operand planes of TDNN5 after a trunk pass that stopped before it
  DevBuf pool_rw, pool_vs, pool_part;           // fused TDNN5 + pooling: row weights, weight sums, per-tile partial sums
  int variant = 0;                     // 0: XVectorSincNet (pyannote/embedding), 1: WeSpeaker ResNet34 (variant B)
  std::unique_ptr<struct ResNet> rn;
};

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
  // work buffers: planes of the waveform, spectrum, log-mel map, three plane pairs per stage, float32 final map
  DevBuf wav_hi, wav_lo, spec, logmel, mean, act[4][3][2], fin;
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
      r.mean.ensure((size_t)U * 80 * 4))
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
  // ---- kaldi fbank: planes of x * 2^15, [rows, 448] x [448, 640] on the tensor cores, power -> mel -> log, time mean
  if ((rc = launch_fb_planes(wav, n, r.wav_hi.p, r.wav_lo.p, st))) return rc;
  {
    TcGemm t{};
    t.A_hi = r.wav_hi.p; t.A_lo = r.wav_lo.p; t.lda = 160; t.Cin = 448; t.KW = 1; t.dil = 1;
    t.Mtot = (long long)U * rpi; t.M = (long long)U * rpi;
    t.N = 640; t.out_f32 = r.spec.as<float>(); t.ldc = 640; t.epi = 0; t.tag = "fbank_dft";
    if ((rc = set_weights(t, r.fb)) || (rc = launch_gemm_tc(t, st))) return rc;
  }
  if ((rc = launch_fb_mel(r.spec.as<float>(), 640, rpi, g.T0, U, r.banks.as<float>(), r.k_lo.as<int>(), r.k_hi.as<int>(),
                          r.logmel.as<float>(), st)) ||
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
static int emb_trunk(dg_emb* h, const float* wav, int U, const Geom& g, cudaStream_t st, int* T_out, bool defer_last,
                     const SincPrep* prep) {
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
  for (int L = 0; L < 5; L++) {
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
  }
  *T_out = T;
  return 0;
}

// TDNN5 (Conv1d(512, 1500, 1) -> LeakyReLU -> BatchNorm) fused with the K weighted statistics poolings: the [rows, 1500] map
// (455 MB at B = 256) is never written; the epilogue leaves per-tile partial sums, pool_finalize turns them into mean / std.
static int emb_tdnn5_pool(dg_emb* h, int U, const Geom& g, const float* weights, int F, int K, int T, float eps,
                          cudaStream_t st) {
  int rc;
  const long long M = (long long)U * g.S2;
  const int m_tiles = (int)((M + 127) / 128);
  if (h->pool_rw.ensure(((size_t)M + 128) * 16) || h->pool_vs.ensure((size_t)U * K * 8) ||
      h->pool_part.ensure((size_t)m_tiles * 2 * 8 * 1500 * 4) || h->pooled.ensure((size_t)U * K * 3000 * 4))
    return DG_ECUDA;
  if ((rc = launch_pool_weights(weights, U, F, K, g.S2, T, h->idx0.as<int>(), h->idx1.as<int>(), h->lam1.as<float>(), eps,
                                h->pool_rw.as<float>(), h->pool_vs.as<float>(), st)))
    return rc;
  TcGemm t{};
  t.A_hi = h->t4h; t.A_lo = h->t4l; t.lda = 512; t.Cin = 512; t.KW = 1; t.dil = 1; t.Mtot = M; t.M = M;
  t.N = 1500; t.bias = h->tb[4].as<float>(); t.bn_scale = h->bns[4].as<float>(); t.bn_shift = h->bnh[4].as<float>();
  t.ldc = 1500; t.epi = 4; t.tag = "tdnn5";
  t.pool_w = h->pool_rw.as<float>(); t.pool_part = h->pool_part.as<float>(); t.pool_item_rows = g.S2; t.pool_K = K;
  if ((rc = set_weights(t, h->tw[4])) || (rc = launch_gemm_tc(t, st))) return rc;
  h->pool_C = 1500;
  return launch_pool_finalize(h->pool_part.as<float>(), h->pool_vs.as<float>(), h->bnh[4].as<float>(), U, K, 1500, g.S2, T, eps,
                              h->pooled.as<float>(), st);
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
static bool pool_fusable(const dg_emb* h, int K, const Geom& g) { return h->variant == 0 && K <= 4 && g.S2 >= 128; }

// Sets g_sm_limit for its lifetime (0: no cap).
struct SmLimit {
  const int prev;
  explicit SmLimit(int limit) : prev(g_sm_limit) { g_sm_limit = limit; }
  ~SmLimit() { g_sm_limit = prev; }
};

// Everything after the embedding trunk: interpolation tables, the K weighted statistics poolings of each item -- fused with
// TDNN5 when `fuse` (the trunk was run with defer_last) -- and the projection, into out [B*K, D].  `sm_cap` caps the grids of
// the fused part (the un-fused pooling and its projection are not capped).
static int emb_tail(dg_emb* h, int B, const Geom& g, const float* weights, int F, int K, int T, bool fuse, int normalize,
                    float norm, float* out, cudaStream_t st, int sm_cap = 0) {
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

// ==================================================================================== clustering
struct dg_cluster {
  int device = 0;
  ClusterParams p;
  DevBuf centers, active, init, prep, prep_d, record;
  DevBuf base, base_active, relabel;   // shared-identity mode: table at the last merge, relabel of created centres
};

extern "C" int dg_cluster_create(int max_speakers, int dim, double tau, double rho, double delta, int device,
                                 dg_cluster** out) {
  if (!out || max_speakers < 1 || max_speakers > 32 || dim < 1) {
    set_error("dg_cluster_create: need 1 <= max_speakers <= 32 and dim >= 1");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_cluster> h(new dg_cluster());
  h->device = device;
  h->p.M = max_speakers;
  h->p.D = dim;
  // numpy compares a float32 array with a Python float in float32 (weak scalar promotion)
  h->p.tau_f = (float)tau;
  h->p.rho_f = (float)rho;
  h->p.delta = delta;
  h->p.metric = 0;
  if (h->centers.ensure((size_t)max_speakers * dim * 8) || h->active.ensure(32 * 4) || h->init.ensure(2 * 4) ||
      h->base.ensure((size_t)max_speakers * dim * 8) || h->base_active.ensure(32 * 4) || h->relabel.ensure(32 * 4))
    return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_cluster_set_metric(dg_cluster* h, int metric) {
  if (!h || metric < 0 || metric > 4) {
    set_error("dg_cluster_set_metric: 0 cosine, 1 euclidean, 2 sqeuclidean, 3 cityblock, 4 chebyshev");
    return DG_EINVAL;
  }
  h->p.metric = metric;
  return DG_OK;
}

extern "C" int dg_cluster_step(dg_cluster* h, const float* seg, const float* emb, int B, int F, int K, int32_t* map,
                               float* permuted, void* stream) {
  if (!h || !seg || !emb || !map || B < 0 || F < 1 || K < 1) {
    set_error("dg_cluster_step: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  if (h->prep.ensure(cluster_prep_floats(B, K) * 4 + 16) || h->prep_d.ensure(cluster_prep_doubles(B, K) * 8 + 16))
    return DG_ECUDA;
  return launch_cluster_step(h->p, seg, emb, B, F, K, h->centers.as<double>(), h->active.as<int>(),
                             h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), map, permuted,
                             (cudaStream_t)stream);
}

extern "C" int dg_cluster_reset(dg_cluster* h) {
  if (!h) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaDeviceSynchronize());
  DG_CUDA(cudaMemset(h->centers.p, 0, h->centers.bytes));
  DG_CUDA(cudaMemset(h->active.p, 0, h->active.bytes));
  DG_CUDA(cudaMemset(h->init.p, 0, h->init.bytes));
  DG_CUDA(cudaMemset(h->base.p, 0, h->base.bytes));
  DG_CUDA(cudaMemset(h->base_active.p, 0, h->base_active.bytes));
  return DG_OK;
}

extern "C" int dg_cluster_get_state(dg_cluster* h, double* centers, int32_t* active, int* initialized) {
  if (!h) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaDeviceSynchronize());
  int init[2] = {0, 0};
  DG_CUDA(cudaMemcpy(init, h->init.p, 8, cudaMemcpyDeviceToHost));
  if (init[1]) {
    set_error("Cannot update unknown centers");   // reference clustering.py:98 (AssertionError)
    return DG_EINVAL;
  }
  if (centers) DG_CUDA(cudaMemcpy(centers, h->centers.p, (size_t)h->p.M * h->p.D * 8, cudaMemcpyDeviceToHost));
  if (active) DG_CUDA(cudaMemcpy(active, h->active.p, (size_t)h->p.M * 4, cudaMemcpyDeviceToHost));
  if (initialized) *initialized = init[0];
  return DG_OK;
}

extern "C" int dg_cluster_set_state(dg_cluster* h, const double* centers, const int32_t* active, int initialized) {
  if (!h || !centers || !active) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaDeviceSynchronize());
  int init[2] = {initialized ? 1 : 0, 0};
  DG_CUDA(cudaMemcpy(h->centers.p, centers, (size_t)h->p.M * h->p.D * 8, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->active.p, active, (size_t)h->p.M * 4, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->init.p, init, 8, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->base.p, centers, (size_t)h->p.M * h->p.D * 8, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->base_active.p, active, (size_t)h->p.M * 4, cudaMemcpyHostToDevice));
  return DG_OK;
}

extern "C" int dg_cluster_destroy(dg_cluster* h) {
  delete h;
  return DG_OK;
}

// shared-identity extension (SURVEY.md 8(e), BASELINE config 5); kernels and rule in cluster.cu
extern "C" int dg_cluster_record_len(const dg_cluster* h) { return h ? h->p.M * h->p.D + h->p.M + 2 : 0; }

extern "C" int dg_cluster_export_delta(dg_cluster* h, double* record_dev, void* stream) {
  if (!h || !record_dev) {
    set_error("dg_cluster_export_delta: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  return launch_cluster_export(h->centers.as<double>(), h->active.as<int>(), h->base.as<double>(),
                               h->base_active.as<int>(), h->p.M, h->p.D, record_dev, (cudaStream_t)stream);
}

extern "C" int dg_cluster_merge(dg_cluster* h, const double* records_dev, int world, int rank, int32_t* maps_dev,
                                int n_maps, void* stream) {
  if (!h || !records_dev || world < 1 || rank < 0 || rank >= world) {
    set_error("dg_cluster_merge: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  int rc;
  if ((rc = launch_cluster_merge(records_dev, world, rank, h->p, dg_cluster_record_len(h), h->centers.as<double>(),
                                 h->active.as<int>(), h->base.as<double>(), h->base_active.as<int>(),
                                 h->init.as<int>(), h->relabel.as<int32_t>(), (cudaStream_t)stream)))
    return rc;
  if (maps_dev && n_maps > 0) return launch_relabel_maps(maps_dev, n_maps, h->relabel.as<int32_t>(), (cudaStream_t)stream);
  return DG_OK;
}

// ================================================================================== self test
extern "C" int dg_selftest_split_f16_host(const float* x, long long n, unsigned short* hi, unsigned short* lo) {
  if (!x || !hi || !lo || n < 0) {
    set_error("dg_selftest_split_f16_host: null argument");
    return DG_EINVAL;
  }
  for (long long i = 0; i < n; i++) {
    hi[i] = host_f32_to_h16(x[i]);
    lo[i] = host_f32_to_h16(x[i] - host_h16_to_f32(hi[i]));
  }
  return DG_OK;
}

// Runs the same shifted-window GEMM through the float32 reference kernel (gemm.cu) and through the wgmma split-precision
// kernel on seeded random data and reports the largest absolute difference and the output scale.
extern "C" int dg_selftest_gemm_tc(int M, int Cin, int KW, int dil, int N, int epi, float* max_abs_diff,
                                   float* out_rms) {
  if (M < 1 || Cin % 64 || KW < 1 || N % 4 || !max_abs_diff || !out_rms) {
    set_error("dg_selftest_gemm_tc: bad arguments");
    return DG_EINVAL;
  }
  const int K = KW * Cin, npad = N == 64 ? 64 : (N + 255) / 256 * 256;
  const long long Mtot = M;
  std::vector<float> A((size_t)Mtot * Cin), Wkn((size_t)K * N), Wnk((size_t)N * K), bias(N), bsc(N), bsh(N);
  uint32_t seed = 12345u;
  auto rnd = [&]() {
    seed = seed * 1664525u + 1013904223u;
    return ((seed >> 8) & 0xFFFF) / 65536.f - 0.5f;
  };
  // DG_SELFTEST_AMP: amplitude of the A operand (default 2): small values put the whole lo plane into fp16's subnormal range
  static const float amp = getenv("DG_SELFTEST_AMP") ? (float)atof(getenv("DG_SELFTEST_AMP")) : 2.f;
  for (auto& v : A) v = amp * rnd();
  for (int k = 0; k < K; k++)
    for (int n = 0; n < N; n++) {
      const float w = rnd() * 0.25f;
      Wkn[(size_t)k * N + n] = w;
      Wnk[(size_t)n * K + k] = w;
    }
  for (int n = 0; n < N; n++) {
    bias[n] = rnd();
    bsc[n] = 1.f + rnd();
    bsh[n] = rnd();
  }
  DevBuf dA, dWkn, dB, dS, dH, dAh, dAl, dC0, dC1, dOh, dOl;
  WeightPlanes dW;
  if (upload(dA, A) || upload(dWkn, Wkn) || upload(dB, bias) || upload(dS, bsc) || upload(dH, bsh) ||
      upload_split(dW, Wnk, N, npad, K))
    return DG_ECUDA;
  if (dAh.ensure((size_t)Mtot * Cin * 2) || dAl.ensure((size_t)Mtot * Cin * 2) || dC0.ensure((size_t)M * N * 4) ||
      dC1.ensure((size_t)M * N * 4) || dOh.ensure((size_t)M * N * 2) || dOl.ensure((size_t)M * N * 2))
    return DG_ECUDA;
  int rc;
  GemmArgs g{};
  g.A = dA.as<float>(); g.lda = Cin; g.Cin = Cin; g.KW = KW; g.dil = dil; g.Mtot = Mtot; g.M = M;
  g.W = dWkn.as<float>(); g.ldw = N; g.N = N; g.bias = dB.as<float>(); g.bn_scale = dS.as<float>();
  g.bn_shift = dH.as<float>(); g.C = dC0.as<float>(); g.ldc = N; g.epi = epi == 0 ? EPI_BIAS : EPI_BIAS_LEAKY_BN;
  g.tag = "selftest_simt";
  if ((rc = launch_gemm(g, nullptr))) return rc;
  if ((rc = launch_split_ex(dA.as<float>(), Mtot, Cin, Cin, Cin, 0, 1, nullptr, nullptr, dAh.p, dAl.p, nullptr))) return rc;
  TcGemm t{};
  t.A_hi = dAh.p; t.A_lo = dAl.p; t.lda = Cin; t.Cin = Cin; t.KW = KW; t.dil = dil; t.Mtot = Mtot; t.M = M;
  t.N = N; t.bias = dB.as<float>(); t.bn_scale = dS.as<float>();
  t.bn_shift = dH.as<float>(); t.out_f32 = dC1.as<float>(); t.out_hi = dOh.p; t.out_lo = dOl.p; t.ldc = N;
  t.epi = epi; t.tag = "selftest_tc";
  if ((rc = set_weights(t, dW)) || (rc = launch_gemm_tc(t, nullptr))) return rc;
  DG_CUDA(cudaDeviceSynchronize());
  std::vector<float> c0((size_t)M * N), c1((size_t)M * N);
  DG_CUDA(cudaMemcpy(c0.data(), dC0.p, c0.size() * 4, cudaMemcpyDeviceToHost));
  std::vector<uint16_t> oh, ol;
  if (epi == 1) {
    oh.resize((size_t)M * N);
    ol.resize((size_t)M * N);
    DG_CUDA(cudaMemcpy(oh.data(), dOh.p, oh.size() * 2, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(ol.data(), dOl.p, ol.size() * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < c1.size(); i++) c1[i] = host_h16_to_f32(oh[i]) + host_h16_to_f32(ol[i]);
  } else {
    DG_CUDA(cudaMemcpy(c1.data(), dC1.p, c1.size() * 4, cudaMemcpyDeviceToHost));
  }
  double md = 0, ss = 0;
  size_t worst = 0, n_big = 0;
  for (size_t i = 0; i < c0.size(); i++) {
    const double d = fabs((double)c0[i] - (double)c1[i]);
    if (!(d <= md)) {     // NaN-propagating max
      md = d;
      worst = i;
    }
    if (!(d <= 1e-2)) n_big++;
    ss += (double)c0[i] * c0[i];
  }
  if (n_big)
    fprintf(stderr, "dg_selftest_gemm_tc: %zu of %zu outputs differ by more than 1e-2; worst at row %zu col %zu: simt %g, wgmma %g\n",
            n_big, c0.size(), worst / N, worst % N, c0[worst], c1[worst]);
  if (n_big && epi == 1) {
    size_t shown = 0;
    for (size_t i = 0; i < c0.size() && shown < 12; i++)
      if (!(fabs((double)c0[i] - (double)c1[i]) <= 1e-2)) {
        fprintf(stderr, "   row %zu col %zu: simt %g, planes hi 0x%04x lo 0x%04x\n", i / N, i % N, c0[i], oh[i], ol[i]);
        shown++;
      }
  }
  *max_abs_diff = (float)md;
  *out_rms = (float)sqrt(ss / c0.size());
  return DG_OK;
}

// ================================================================================ fused pipeline
// Persistent worker threads for the host-side gather of dg_pipeline_call_host (B separate pageable windows -> pinned staging):
// created once per pipeline handle; a job is one callable that every worker runs concurrently (the callable hands out work
// items through its own atomic counter).
class GatherPool {
 public:
  explicit GatherPool(int n) {
    for (int i = 0; i < n; i++) th_.emplace_back([this] { loop(); });
  }
  ~GatherPool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  int size() const { return (int)th_.size(); }
  void start(std::function<void()> fn) {       // returns at once; wait() returns when every worker has finished fn
    {
      std::lock_guard<std::mutex> lk(mu_);
      job_ = std::move(fn);
      generation_++;
      active_ = (int)th_.size();
    }
    cv_.notify_all();
  }
  void wait() {
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [this] { return active_ == 0; });
  }

 private:
  void loop() {
    int seen = 0;
    for (;;) {
      std::function<void()> fn;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return stop_ || generation_ != seen; });
        if (stop_) return;
        seen = generation_;
        fn = job_;
      }
      fn();
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (--active_ == 0) done_.notify_all();
      }
    }
  }
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  std::function<void()> job_;
  int generation_ = 0, active_ = 0;
  bool stop_ = false;
};

// a step's outputs: scores [B, F, K], embeddings [B, K, D], speaker maps [B, K], permuted scores [B, F, M]
struct StepShape {
  int B = 0, F = 0, K = 0;
  size_t seg_bytes() const { return (size_t)B * F * K * 4; }
  size_t emb_bytes(int D) const { return (size_t)B * K * D * 4; }
  size_t map_bytes() const { return (size_t)B * K * 4; }
  size_t permuted_bytes(int M) const { return (size_t)B * F * M * 4; }
};
struct StepOut { float *seg, *emb; int32_t* map; float* permuted; };   // where a step's outputs are or go; null: not wanted

struct dg_pipeline {
  dg_seg* seg;
  dg_emb* emb;
  dg_cluster* clu;
  float gamma, beta;
  int normalize_weights;
  int hop = 0;          // samples between consecutive windows of a batch (hint, dg_pipeline_set_hop); 0 = unknown
  // Members are destroyed in reverse order: the streams and events (declared last) first, then the pinned staging, then
  // the device buffers and worker threads.
  DevBuf wav, segd, embd, mapd, permd, osp[2];
  SincPrep prep[2];
  // Every step runs through pipeline_enqueue.  Submitted step n (up to DG_MAX_INFLIGHT outstanding) uses result / input slot
  // n % 3 and scratch lane n & 1: two steps compute concurrently while the host uploads step n+2.  Synchronous steps use lane
  // 0 and the caller's buffers or wav / segd / ..., never a slot (collected pointers stay valid), and do not count in next_step.
  DevBuf slot_wav[3], slot_seg[3], slot_emb[3], slot_map[3];
  StepShape slot_shape[3];
  int outstanding = 0;
  long long next_step = 0;
  long long ident_merged_upto = 0;      // steps below this index have had their maps relabelled by a merge
  std::unique_ptr<GatherPool> gather;   // worker threads of the host gather (created at the first dg_pipeline_call_host)
  DevBuf call_stream;                   // device image of the stream a dg_pipeline_call_host batch was cut from
  long long call_h2d_bytes = 0;         // bytes the last dg_pipeline_call_host uploaded
  PinnedBuf pin_wav;                    // pinned staging of dg_pipeline_call_host (B separate host windows -> one upload)
  Stream st;
  // two-stream overlap inside a step: the segmentation chain (critical path, high priority) and the
  // embedding trunk (independent of it until the pooling weights exist) run concurrently
  Stream s_seg[2], s_emb, s_clu, s_h2d, s_d2h;
  Event e_osp[2], e_prep[2], e_start, e_emb, e_done;
  Event e_h2d[3], e_slot_done[3], e_lane_done[2];
  // shared-identity mode inside the pipelined flow: export / merge run on the clustering stream, in order with the clustering
  // of the submitted steps, so the networks of the next steps keep running meanwhile (created at the first export)
  Event e_ident, e_ident_in;
  StepOut slot_out(int s) const { return {slot_seg[s].as<float>(), slot_emb[s].as<float>(), slot_map[s].as<int32_t>()}; }
};

extern "C" int dg_pipeline_create(dg_seg* seg, dg_emb* emb, dg_cluster* clu, float gamma, float beta,
                                  int normalize_weights, dg_pipeline** out) {
  if (!seg || !emb || !clu || !out) {
    set_error("dg_pipeline_create: null handle");
    return DG_EINVAL;
  }
  if (seg->device != emb->device || seg->device != clu->device) {
    set_error("dg_pipeline_create: handles live on different devices");
    return DG_EINVAL;
  }
  if (clu->p.D != emb->D) {
    set_error("dg_pipeline_create: clustering dimension != embedding dimension");
    return DG_EINVAL;
  }
  std::unique_ptr<dg_pipeline> h(new dg_pipeline());
  h->seg = seg; h->emb = emb; h->clu = clu;
  h->gamma = gamma; h->beta = beta; h->normalize_weights = normalize_weights;
  DG_CUDA(cudaSetDevice(seg->device));
  int lo = 0, hi = 0;
  DG_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  if (h->st.create() || h->s_seg[0].create(hi) || h->s_emb.create(lo) || h->s_clu.create(hi) || h->s_seg[1].create(hi) ||
      h->s_h2d.create() || h->s_d2h.create())
    return DG_ECUDA;
  for (Event* e : {&h->e_start, &h->e_osp[0], &h->e_emb, &h->e_done, &h->e_osp[1], &h->e_prep[0], &h->e_prep[1], &h->e_h2d[0],
                   &h->e_h2d[1], &h->e_h2d[2], &h->e_slot_done[0], &h->e_slot_done[1], &h->e_slot_done[2],
                   &h->e_lane_done[0], &h->e_lane_done[1]})
    if (e->create()) return DG_ECUDA;
  DG_CUDA(cudaEventRecord(h->e_emb, h->s_emb));   // so that the first step's wait on it is well defined
  *out = h.release();
  return DG_OK;
}

// DG_CALL_TIMING=1: device time stamps of the sub-batches of dg_pipeline_call_host (diagnostic)
struct CallDiag {
  cudaEvent_t t0 = nullptr, up[3], prep[3], trunk[3], seg[3], emb[3], clu[3];
  int j = 0;
  void create() {
    if (t0) return;
    cudaEventCreate(&t0);
    for (int i = 0; i < 3; i++)
      for (cudaEvent_t* e : {&up[i], &prep[i], &trunk[i], &seg[i], &emb[i], &clu[i]}) cudaEventCreate(e);
  }
};
static thread_local CallDiag* g_diag = nullptr;
#define DG_DIAG(field, stream)                                        \
  do {                                                                \
    if (g_diag) cudaEventRecord(g_diag->field[g_diag->j], stream);    \
  } while (0)

// grid cap of the embedding stream's persistent kernels while the segmentation stream runs a recurrence over B windows: the
// SMs the recurrence leaves free, or no cap if that would be half of the device or less
static int emb_sm_cap(int device, int B) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int lstm_ctas = lstm_tc_ctas(B);
  return sms - lstm_ctas > sms / 2 ? sms - lstm_ctas : 0;
}

// segmentation chain on s_seg and embedding chain on s_emb, both starting after `start`; on return
// e_emb (recorded on s_emb) marks seg, osp and emb complete
static int pipeline_nets(dg_pipeline* h, const float* wav, int S, const StepShape& sh, float* seg, float* emb,
                         cudaEvent_t start, int lane, int stream_hop) {
  int rc;
  const int B = sh.B, F = sh.F, K = sh.K;
  const Geom g = make_geom(S);
  // lane 0 / 1: segmentation stream, scratch set, OSP buffer and event of this step (consecutive pipelined steps
  // alternate, so step i+1's segmentation chain can start while step i's is still in its recurrence)
  cudaStream_t s_seg = h->s_seg[lane];
  DevBuf& osp = h->osp[lane];
  if (osp.ensure(sh.seg_bytes())) return DG_ECUDA;
  DG_CUDA(cudaStreamWaitEvent(s_seg, start, 0));
  DG_CUDA(cudaStreamWaitEvent(h->s_emb, start, 0));
  // another pipeline (or a block-level call) that used these model handles' scratch last: stream-ordered hand-over
  LaneUse seg_use(h->seg->guard[lane], h, s_seg), emb_use(h->emb->guard, h, h->s_emb);
  if ((rc = seg_use.rc) || (rc = emb_use.rc)) return rc;
  // waveform statistics + standardised fp16 planes once, for both networks' SincNets
  SincPrep& prep = h->prep[lane];
  if ((rc = run_sinc_prep(prep, wav, B, g, s_seg, stream_hop ? stream_hop : h->hop, stream_hop != 0))) return rc;
  DG_CUDA(cudaEventRecord(h->e_prep[lane], s_seg));
  DG_DIAG(prep, s_seg);
  DG_CUDA(cudaStreamWaitEvent(h->s_emb, h->e_prep[lane], 0));
  // embedding trunk first in host order (low-priority stream, grid capped to the SMs the LSTM leaves free)
  int T = 0;
  const bool fuse = pool_fusable(h->emb, K, g);
  const int sm_cap = emb_sm_cap(h->seg->device, B);
  {
    SmLimit cap(sm_cap);
    if ((rc = emb_trunk(h->emb, wav, B, g, h->s_emb, &T, fuse, &prep))) return rc;
  }
  DG_DIAG(trunk, h->s_emb);
  if ((rc = seg_forward_lane(h->seg, lane, &prep, wav, B, S, seg, s_seg))) return rc;
  if ((rc = dg_osp(seg, B, F, K, h->gamma, h->beta, h->normalize_weights, osp.as<float>(), s_seg))) return rc;
  DG_CUDA(cudaEventRecord(h->e_osp[lane], s_seg));
  if ((rc = seg_use.end())) return rc;
  DG_DIAG(seg, s_seg);
  DG_CUDA(cudaStreamWaitEvent(h->s_emb, h->e_osp[lane], 0));
  // a fused TDNN5 needs the pooling weights: it runs here, after the segmentation of this step, with its grid capped like the
  // trunk's (the other lane's recurrence may hold 2 x ceil(B/16) SMs at this point)
  if ((rc = emb_tail(h->emb, B, g, osp.as<float>(), F, K, T, fuse, 1, 1.f, emb, h->s_emb, sm_cap))) return rc;
  DG_CUDA(cudaEventRecord(h->e_emb, h->s_emb));
  DG_DIAG(emb, h->s_emb);
  return emb_use.end();
}

extern "C" int dg_pipeline_set_hop(dg_pipeline* h, int hop_samples) {
  if (!h || hop_samples < 0) {
    set_error("dg_pipeline_set_hop: bad arguments");
    return DG_EINVAL;
  }
  h->hop = hop_samples;
  return DG_OK;
}

// Enqueues one step: networks on scratch lane `lane` after `start`, clustering on s_clu, outputs to `out`.  stream_hop > 0:
// the batch was cut on the device from one stream, windows that many samples apart (sinc layer in stream form, no overlap
// check).  slot >= 0: a submitted step in that result slot, marked clustered by e_slot_done[slot]; else by e_done.
static int pipeline_enqueue(dg_pipeline* h, const float* wav, int S, const StepShape& sh, int lane, cudaEvent_t start,
                            int stream_hop, const StepOut& out, int slot) {
  int rc;
  // the slot's previous occupant (three submits ago) must be fully clustered, and the lane's previous user past its
  // embeddings, before their buffers are rewritten
  for (cudaStream_t s : {(cudaStream_t)h->s_seg[lane], (cudaStream_t)h->s_emb}) {
    if (slot >= 0) DG_CUDA(cudaStreamWaitEvent(s, h->e_slot_done[slot], 0));
    DG_CUDA(cudaStreamWaitEvent(s, h->e_lane_done[lane], 0));
  }
  if ((rc = pipeline_nets(h, wav, S, sh, out.seg, out.emb, start, lane, stream_hop))) return rc;
  // the lane's scratch (waveform planes, segmentation activations, OSP weights) is free as soon as this step's embeddings
  // exist -- the clustering reads only the step's outputs -- so the step after next may start before this one is clustered
  DG_CUDA(cudaEventRecord(h->e_lane_done[lane], h->s_emb));
  DG_CUDA(cudaStreamWaitEvent(h->s_clu, h->e_emb, 0));
  if ((rc = dg_cluster_step(h->clu, out.seg, out.emb, sh.B, sh.F, sh.K, out.map, out.permuted, h->s_clu))) return rc;
  DG_CUDA(cudaEventRecord(slot >= 0 ? h->e_slot_done[slot] : h->e_done, h->s_clu));
  DG_DIAG(clu, h->s_clu);
  return DG_OK;
}

// a synchronous step: lane 0, no slot; `st` waits for its clustering
static int pipeline_step(dg_pipeline* h, const float* wav, int S, const StepShape& sh, const StepOut& out, cudaStream_t st,
                         int stream_hop) {
  int rc;
  // DG_NO_OVERLAP=1 (diagnostic): the networks and the clustering back to back on `st`, for kernel-alone timings
  static const bool serial = getenv("DG_NO_OVERLAP") && getenv("DG_NO_OVERLAP")[0] == '1';
  if (serial) {
    if (h->osp[0].ensure(sh.seg_bytes())) return DG_ECUDA;
    if ((rc = dg_seg_forward(h->seg, wav, sh.B, S, out.seg, st))) return rc;
    if ((rc = dg_osp(out.seg, sh.B, sh.F, sh.K, h->gamma, h->beta, h->normalize_weights, h->osp[0].as<float>(), st))) return rc;
    if ((rc = dg_emb_forward(h->emb, wav, h->osp[0].as<float>(), sh.B, S, sh.F, sh.K, 1, 1.f, out.emb, st))) return rc;
    return dg_cluster_step(h->clu, out.seg, out.emb, sh.B, sh.F, sh.K, out.map, out.permuted, st);
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  DG_CUDA(cudaEventRecord(h->e_start, st));
  if ((rc = pipeline_enqueue(h, wav, S, sh, 0, h->e_start, stream_hop, out, -1))) return rc;
  DG_CUDA(cudaStreamWaitEvent(st, h->e_done, 0));
  return DG_OK;
}

// `st` waits for `done` (if any), then copies the outputs of a step of shape `sh` from `src` to the non-null members of `dst`
static int copy_out(const dg_pipeline* h, cudaStream_t st, cudaEvent_t done, const StepShape& sh, const StepOut& src,
                    const StepOut& dst, cudaMemcpyKind kind) {
  if (done) DG_CUDA(cudaStreamWaitEvent(st, done, 0));
  if (dst.seg) DG_CUDA(cudaMemcpyAsync(dst.seg, src.seg, sh.seg_bytes(), kind, st));
  if (dst.emb) DG_CUDA(cudaMemcpyAsync(dst.emb, src.emb, sh.emb_bytes(h->emb->D), kind, st));
  if (dst.map) DG_CUDA(cudaMemcpyAsync(dst.map, src.map, sh.map_bytes(), kind, st));
  if (dst.permuted) DG_CUDA(cudaMemcpyAsync(dst.permuted, src.permuted, sh.permuted_bytes(h->clu->p.M), kind, st));
  return DG_OK;
}

extern "C" int dg_pipeline_step(dg_pipeline* h, const float* wav, int B, int S, float* seg, float* emb, int32_t* map,
                                float* permuted, void* stream) {
  if (!h || !wav || !seg || !emb || !map || B < 1) {
    set_error("dg_pipeline_step: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error("dg_pipeline_step: submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  return pipeline_step(h, wav, S, {B, F, K}, {seg, emb, map, permuted}, (cudaStream_t)stream, 0);
}

// ---- pipelined variants (up to three steps outstanding, two computing): the sequential clustering of step i and the host copies overlap the
//      networks of step i+1.  Per stream the chunk order is preserved: clustering runs on one stream.
static const int DG_MAX_INFLIGHT = 3;

// enqueues submitted step next_step (result slot next_step % 3, lane next_step & 1) and books it outstanding
static int pipeline_submit(dg_pipeline* h, const float* wav, int S, const StepShape& sh, cudaEvent_t start, int stream_hop) {
  int rc;
  const int slot = (int)(h->next_step % 3);
  if (h->slot_seg[slot].ensure(sh.seg_bytes()) || h->slot_emb[slot].ensure(sh.emb_bytes(h->emb->D)) ||
      h->slot_map[slot].ensure(sh.map_bytes()))
    return DG_ECUDA;
  if ((rc = pipeline_enqueue(h, wav, S, sh, (int)(h->next_step & 1), start, stream_hop, h->slot_out(slot), slot))) return rc;
  h->slot_shape[slot] = sh;
  h->next_step++;
  h->outstanding++;
  return DG_OK;
}

extern "C" int dg_pipeline_submit(dg_pipeline* h, const float* wav_dev, int B, int S, void* stream) {
  if (!h || !wav_dev || B < 1) {
    set_error("dg_pipeline_submit: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding >= DG_MAX_INFLIGHT) {
    set_error("dg_pipeline_submit: three steps are already outstanding; collect one first");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  DG_CUDA(cudaEventRecord(h->e_start, (cudaStream_t)stream));
  return pipeline_submit(h, wav_dev, S, {B, F, K}, h->e_start, 0);
}

extern "C" int dg_pipeline_collect(dg_pipeline* h, const float** seg_dev, const float** emb_dev,
                                   const int32_t** map_dev, void* stream) {
  if (!h || h->outstanding < 1) {
    set_error("dg_pipeline_collect: nothing outstanding");
    return DG_EINVAL;
  }
  const int slot = (int)((h->next_step - h->outstanding) % 3);
  DG_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->e_slot_done[slot], 0));
  if (seg_dev) *seg_dev = h->slot_seg[slot].as<float>();
  if (emb_dev) *emb_dev = h->slot_emb[slot].as<float>();
  if (map_dev) *map_dev = h->slot_map[slot].as<int32_t>();
  h->outstanding--;
  return DG_OK;
}

extern "C" int dg_pipeline_collect_copy(dg_pipeline* h, float* seg_dev, float* emb_dev, int32_t* map_dev,
                                        void* stream) {
  if (!h || h->outstanding < 1) {
    set_error("dg_pipeline_collect_copy: nothing outstanding");
    return DG_EINVAL;
  }
  const int slot = (int)((h->next_step - h->outstanding) % 3);
  const int rc = copy_out(h, (cudaStream_t)stream, h->e_slot_done[slot], h->slot_shape[slot], h->slot_out(slot),
                          {seg_dev, emb_dev, map_dev, nullptr}, cudaMemcpyDeviceToDevice);
  if (rc) return rc;
  h->outstanding--;
  return DG_OK;
}

extern "C" int dg_pipeline_submit_host(dg_pipeline* h, const float* wav_host, int B, int S) {
  if (!h || !wav_host || B < 1) {
    set_error("dg_pipeline_submit_host: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding >= DG_MAX_INFLIGHT) {
    set_error("dg_pipeline_submit_host: three steps are already outstanding; collect one first");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  const int slot = (int)(h->next_step % 3);
  if (h->slot_wav[slot].ensure((size_t)B * S * 4)) return DG_ECUDA;
  DG_CUDA(cudaStreamWaitEvent(h->s_h2d, h->e_slot_done[slot], 0));
  DG_CUDA(cudaMemcpyAsync(h->slot_wav[slot].p, wav_host, (size_t)B * S * 4, cudaMemcpyHostToDevice, h->s_h2d));
  DG_CUDA(cudaEventRecord(h->e_h2d[slot], h->s_h2d));
  return pipeline_submit(h, h->slot_wav[slot].as<float>(), S, {B, F, K}, h->e_h2d[slot], 0);
}

extern "C" int dg_pipeline_collect_host(dg_pipeline* h, float* seg_host, float* emb_host, int32_t* map_host) {
  if (!h || h->outstanding < 1) {
    set_error("dg_pipeline_collect_host: nothing outstanding");
    return DG_EINVAL;
  }
  const int slot = (int)((h->next_step - h->outstanding) % 3);
  const int rc = copy_out(h, h->s_d2h, h->e_slot_done[slot], h->slot_shape[slot], h->slot_out(slot),
                          {seg_host, emb_host, map_host, nullptr}, cudaMemcpyDeviceToHost);
  if (rc) return rc;
  DG_CUDA(cudaStreamSynchronize(h->s_d2h));
  h->outstanding--;
  return DG_OK;
}

extern "C" int dg_pipeline_step_host(dg_pipeline* h, const float* wav_host, int B, int S, float* seg_host,
                                     float* emb_host, int32_t* map_host, float* permuted_host) {
  if (!h || !wav_host || B < 1) {
    set_error("dg_pipeline_step_host: bad arguments");
    return DG_EINVAL;
  }
  int rc;
  StepShape sh = {B};
  if ((rc = dg_seg_dims(h->seg, S, &sh.F, &sh.K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  if (h->wav.ensure((size_t)B * S * 4) || h->segd.ensure(sh.seg_bytes()) || h->embd.ensure(sh.emb_bytes(h->emb->D)) ||
      h->mapd.ensure(sh.map_bytes()) || (permuted_host && h->permd.ensure(sh.permuted_bytes(h->clu->p.M))))
    return DG_ECUDA;
  DG_CUDA(cudaMemcpyAsync(h->wav.p, wav_host, (size_t)B * S * 4, cudaMemcpyHostToDevice, h->st));
  const StepOut dev = {h->segd.as<float>(), h->embd.as<float>(), h->mapd.as<int32_t>(),
                       permuted_host ? h->permd.as<float>() : nullptr};
  if ((rc = dg_pipeline_step(h, h->wav.as<float>(), B, S, dev.seg, dev.emb, dev.map, dev.permuted, h->st))) return rc;
  if ((rc = copy_out(h, h->st, nullptr, sh, dev, {seg_host, emb_host, map_host, permuted_host}, cudaMemcpyDeviceToHost)))
    return rc;
  DG_CUDA(cudaStreamSynchronize(h->st));
  return DG_OK;
}

// ======================================================================== resampling
// torchaudio's T.Resample(orig, new) with its defaults (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99) -- what the
// reference's blocks.Resample applies to every window of a source at another rate (reference blocks/utils.py:62-89).  The taps
// come from the host (diart_b200.operators.sinc_resample_kernel), bit-identical to torchaudio's.
struct dg_resample {
  int device = 0;
  RsGeom g{};
  DevBuf taps;   // [n][T]
};

extern "C" int dg_resample_create(int orig, int new_rate, const float* kernel_host, int width, int device, dg_resample** out) {
  if (!out || !kernel_host || orig < 1 || new_rate < 1 || orig == new_rate) {
    set_error("dg_resample_create: rates must be positive and different, taps non-null");
    return DG_EINVAL;
  }
  const int gcd = std::gcd(orig, new_rate);
  RsGeom g;
  g.o = orig / gcd;
  g.n = new_rate / gcd;
  // torchaudio: width = ceil(lowpass_filter_width * orig / (min(orig, new) * rolloff)) on the reduced rates
  const double base = std::min(g.o, g.n) * 0.99;
  const int want = (int)std::ceil(6.0 * g.o / base);
  if (width != want) {
    set_error("dg_resample_create: taps of shape (" + std::to_string(g.n) + ", " + std::to_string(2 * width + g.o) +
              ") given, (" + std::to_string(g.n) + ", " + std::to_string(2 * want + g.o) + ") expected for " +
              std::to_string(orig) + " -> " + std::to_string(new_rate) + " Hz");
    return DG_EINVAL;
  }
  g.w = width;
  g.T = 2 * width + g.o;
  if (!resample_geom_ok(g)) {
    set_error("dg_resample_create: the reduced rate ratio " + std::to_string(g.o) + " / " + std::to_string(g.n) +
              " is too large for the resampling kernel");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_resample> h(new dg_resample());
  h->device = device;
  h->g = g;
  if (h->taps.ensure((size_t)g.n * g.T * 4)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->taps.p, kernel_host, (size_t)g.n * g.T * 4, cudaMemcpyHostToDevice));
  *out = h.release();
  return DG_OK;
}

extern "C" int64_t dg_resample_out_len(const dg_resample* h, int64_t num_samples) {
  if (!h || num_samples < 0) return -1;
  return resample_out_len(h->g, num_samples);
}

extern "C" int dg_resample_forward(dg_resample* h, const float* in_dev, int B, int64_t L, float* out_dev, void* stream) {
  if (!h || !in_dev || !out_dev || B < 1 || L < 1) {
    set_error("dg_resample_forward: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  const long long out_len = resample_out_len(h->g, L);
  RsJob j{};
  j.x = in_dev;
  j.base = RsItem{0, L, 0, out_len, 0};
  j.start_step = L;
  j.out_step = out_len;
  j.W = h->taps.as<float>();
  j.g = h->g;
  j.out = out_dev;
  return launch_resample(j, B, out_len, (cudaStream_t)stream);
}

extern "C" int dg_resample_destroy(dg_resample* h) {
  delete h;
  return DG_OK;
}

// ======================================================================== device-side audio stream
// rearrange_audio_stream (reference src/diart/operators.py:44-100) on the device: the host pushes each sample ONCE
// (8 000 new samples per chunk instead of the 80 000 of a stacked window: 8.2 MB instead of 82 MB per 256-chunk step),
// windows are formed from a circular ring in HBM.
struct dg_stream {
  int device = 0, S = 0, hop = 0, C = 0;   // S, hop, C and the counters are in samples at the source rate
  long long wpos = 0, rpos = 0;          // absolute sample counters: pushed / start of the next window
  dg_resample* rs = nullptr;             // borrowed; windows are resampled to rs's rate (dg_stream_create_resampled)
  DevBuf ring, ys, crop_items, crop_out; // ys: stream-form outputs of the last batch; crop_*: dg_stream_crop_host
  PinnedBuf crop_pin;
  PinnedBuf pin;                         // pinned mirror of the ring (staging for the uploads)
  Stream st;                             // uploads
  Event e_up, e_read;
  // uploads still reading the pinned mirror: (first absolute sample, event); a region of the mirror is rewritten only
  // after the upload that last used it has completed
  std::deque<std::pair<long long, Event>> inflight;
  std::vector<Event> spare;
};

extern "C" int dg_stream_create(int chunk_samples, int step_samples, int max_windows, int device, dg_stream** out) {
  if (!out || chunk_samples < 4 || step_samples < 4 || chunk_samples % 4 || step_samples % 4 || max_windows < 1 ||
      step_samples > chunk_samples) {
    set_error("dg_stream_create: chunk and step must be positive multiples of 4 samples, step <= chunk");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_stream> h(new dg_stream());
  h->device = device; h->S = chunk_samples; h->hop = step_samples;
  // room for the windows being read, a full batch being uploaded meanwhile, and the overlap tail
  h->C = ((chunk_samples + 2 * max_windows * step_samples + 1023) / 1024) * 1024;
  if (h->ring.ensure((size_t)h->C * 4) || h->pin.ensure((size_t)h->C * 4) || h->st.create() || h->e_up.create() ||
      h->e_read.create())
    return DG_ECUDA;
  DG_CUDA(cudaEventRecord(h->e_read, h->st));
  *out = h.release();
  return DG_OK;
}

// the same stream with its windows resampled by `rs` (borrowed): chunk and step count source-rate samples, in any number;
// dg_stream_windows returns [B, dg_resample_out_len(rs, chunk)] resampled windows
extern "C" int dg_stream_create_resampled(int chunk_samples, int step_samples, dg_resample* rs, int max_windows, int device,
                                          dg_stream** out) {
  if (!out || !rs || chunk_samples < 1 || step_samples < 1 || max_windows < 1 || step_samples > chunk_samples ||
      rs->device != device || resample_out_len(rs->g, chunk_samples) > (1 << 30)) {
    set_error("dg_stream_create_resampled: chunk and step must be positive, step <= chunk, resampler on the same device");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_stream> h(new dg_stream());
  h->device = device; h->S = chunk_samples; h->hop = step_samples; h->rs = rs;
  h->C = ((chunk_samples + 2 * max_windows * step_samples + 1023) / 1024) * 1024;
  if (h->ring.ensure((size_t)h->C * 4) || h->pin.ensure((size_t)h->C * 4) || h->st.create() || h->e_up.create() ||
      h->e_read.create())
    return DG_ECUDA;
  DG_CUDA(cudaEventRecord(h->e_read, h->st));
  *out = h.release();
  return DG_OK;
}

// samples per window as dg_stream_windows returns them
static int stream_window_len(const dg_stream* h) { return h->rs ? (int)resample_out_len(h->rs->g, h->S) : h->S; }

extern "C" int dg_stream_destroy(dg_stream* h) {
  delete h;
  return DG_OK;
}

extern "C" int dg_stream_reset(dg_stream* h) {
  if (!h) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaStreamSynchronize(h->st));
  h->wpos = h->rpos = 0;
  for (auto& e : h->inflight) h->spare.push_back(std::move(e.second));
  h->inflight.clear();
  return DG_OK;
}

// complete windows that have been pushed but not yet consumed
extern "C" int dg_stream_available(const dg_stream* h) {
  if (!h) return 0;
  const long long have = h->wpos - h->rpos;
  return have < h->S ? 0 : (int)((have - h->S) / h->hop + 1);
}

// appends n samples (host memory, any kind) to the stream; returns once they are staged (the upload is asynchronous)
extern "C" int dg_stream_push_host(dg_stream* h, const float* samples, int n) {
  if (!h || !samples || n < 0) {
    set_error("dg_stream_push_host: bad arguments");
    return DG_EINVAL;
  }
  if (h->wpos + n - h->rpos > h->C) {
    set_error("dg_stream_push_host: ring full (" + std::to_string(h->wpos - h->rpos) + " samples buffered, capacity " +
              std::to_string(h->C) + "): consume windows first");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  // samples older than rpos may be overwritten: uploads are ordered after the last kernel that read the ring
  DG_CUDA(cudaStreamWaitEvent(h->st, h->e_read, 0));
  // the mirror region [wpos, wpos + n) was last used by the uploads of samples one lap earlier: wait for those
  while (!h->inflight.empty() && h->inflight.front().first < h->wpos + n - h->C) {
    DG_CUDA(cudaEventSynchronize(h->inflight.front().second));
    h->spare.push_back(std::move(h->inflight.front().second));
    h->inflight.pop_front();
  }
  float* pin = h->pin.as<float>();
  int done = 0;
  while (done < n) {
    const int at = (int)((h->wpos + done) % h->C);
    const int len = std::min(n - done, h->C - at);
    memcpy(pin + at, samples + done, (size_t)len * 4);
    DG_CUDA(cudaMemcpyAsync(h->ring.as<float>() + at, pin + at, (size_t)len * 4, cudaMemcpyHostToDevice, h->st));
    done += len;
  }
  Event ev;
  if (!h->spare.empty()) {
    ev = std::move(h->spare.back());
    h->spare.pop_back();
  } else if (ev.create()) {
    return DG_ECUDA;
  }
  DG_CUDA(cudaEventRecord(ev, h->st));
  h->inflight.emplace_back(h->wpos, std::move(ev));
  h->wpos += n;
  DG_CUDA(cudaEventRecord(h->e_up, h->st));
  return DG_OK;
}

// materialises the next B windows as a dense [B, S] batch on `st` and advances the stream by B steps
static int stream_expand(dg_stream* h, int B, float* wav_dev, cudaStream_t st) {
  if (dg_stream_available(h) < B) {
    set_error("dg_stream: " + std::to_string(B) + " windows requested, " + std::to_string(dg_stream_available(h)) + " available");
    return DG_EINVAL;
  }
  DG_CUDA(cudaStreamWaitEvent(st, h->e_up, 0));
  int rc;
  if (h->rs) {
    const RsGeom& g = h->rs->g;
    const long long out_len = resample_out_len(g, h->S);
    // ys is rewritten: the previous batch, possibly formed on another stream, must have been read
    DG_CUDA(cudaStreamWaitEvent(st, h->e_read, 0));
    if (h->hop % g.o == 0) {   // stream form: window b's inner outputs are the stream's outputs
      const long long nr = (long long)(B - 1) * (h->hop / g.o) + (out_len + g.n - 1) / g.n;
      if (h->ys.ensure((size_t)nr * g.n * 4)) return DG_ECUDA;
      if ((rc = launch_resample_stream(h->ring.as<float>(), h->C, h->rpos, h->hop, h->S, B, h->rs->taps.as<float>(), g,
                                       h->ys.as<float>(), wav_dev, st)))
        return rc;
    } else {                   // per-window form, straight from the ring
      RsJob j{};
      j.x = h->ring.as<float>();
      j.C = h->C;
      j.base = RsItem{h->rpos, h->S, 0, out_len, 0};
      j.start_step = h->hop;
      j.out_step = out_len;
      j.W = h->rs->taps.as<float>();
      j.g = g;
      j.out = wav_dev;
      if ((rc = launch_resample(j, B, out_len, st))) return rc;
    }
  } else {
    if (h->rpos % 4) {
      set_error("dg_stream: window start is not 16-byte aligned");
      return DG_EINVAL;
    }
    if ((rc = launch_expand_windows(h->ring.as<float>(), h->rpos, h->C, h->hop, h->S, B, wav_dev, st))) return rc;
  }
  DG_CUDA(cudaEventRecord(h->e_read, st));
  h->rpos += (long long)B * h->hop;
  return 0;
}

extern "C" int dg_stream_windows(dg_stream* h, int B, float* wav_dev, void* stream) {
  if (!h || !wav_dev || B < 1) {
    set_error("dg_stream_windows: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  return stream_expand(h, B, wav_dev, (cudaStream_t)stream);
}

// outputs [first, first + count) of resampled window `window` (counted from the stream's start or last reset), for n
// ranges {window, first, count}, packed into out_host; the window's source samples must still be in the ring.  Every output
// is computed as in dg_stream_windows, so the values are bit-identical to the windows'.  Synchronous.
extern "C" int dg_stream_crop_host(dg_stream* h, int n, const int64_t* ranges_host, float* out_host) {
  if (!h || !h->rs || n < 0 || (n && (!ranges_host || !out_host))) {
    set_error("dg_stream_crop_host: bad arguments (a resampled stream is required)");
    return DG_EINVAL;
  }
  if (!n) return DG_OK;
  const long long out_len = resample_out_len(h->rs->g, h->S);
  std::vector<RsItem> items((size_t)n);
  long long total = 0, max_cnt = 1;
  for (int i = 0; i < n; ++i) {
    const long long win = ranges_host[3 * i], lo = ranges_host[3 * i + 1], cnt = ranges_host[3 * i + 2];
    const long long start = win * h->hop;
    if (win < 0 || lo < 0 || cnt < 0 || lo + cnt > out_len) {
      set_error("dg_stream_crop_host: range " + std::to_string(i) + " lies outside the window");
      return DG_EINVAL;
    }
    if (start < h->wpos - h->C || start + h->S > h->wpos) {
      set_error("dg_stream_crop_host: window " + std::to_string(win) + " is not (or no longer) in the ring");
      return DG_EINVAL;
    }
    items[i] = RsItem{start, h->S, lo, cnt, total};
    total += cnt;
    max_cnt = std::max(max_cnt, cnt);
  }
  DG_CUDA(cudaSetDevice(h->device));
  if (h->crop_items.ensure(items.size() * sizeof(RsItem)) || h->crop_out.ensure((size_t)std::max(total, 1LL) * 4) ||
      h->crop_pin.ensure(std::max(items.size() * sizeof(RsItem), (size_t)total * 4)))
    return DG_ECUDA;
  memcpy(h->crop_pin.h, items.data(), items.size() * sizeof(RsItem));
  DG_CUDA(cudaMemcpyAsync(h->crop_items.p, h->crop_pin.h, items.size() * sizeof(RsItem), cudaMemcpyHostToDevice, h->st));
  RsJob j{};
  j.x = h->ring.as<float>();
  j.C = h->C;
  j.items = h->crop_items.as<RsItem>();
  j.W = h->rs->taps.as<float>();
  j.g = h->rs->g;
  j.out = h->crop_out.as<float>();
  int rc;
  if ((rc = launch_resample(j, n, max_cnt, h->st))) return rc;
  DG_CUDA(cudaMemcpyAsync(h->crop_pin.h, h->crop_out.p, (size_t)total * 4, cudaMemcpyDeviceToHost, h->st));
  DG_CUDA(cudaStreamSynchronize(h->st));
  memcpy(out_host, h->crop_pin.h, (size_t)total * 4);
  return DG_OK;
}

// =============================================================================== device post-path
// DelayedAggregation (hamming, loose) + Binarize of reference diarization.py:205-232 on the device (post.cu).  The handle keeps
// the scores and speaker maps of the last `num_windows - 1` chunks (the reference's pred_buffer) on the device.
struct dg_post {
  int device = 0, F = 0, K = 0, M = 0, nw = 1;
  double tau = 0.5;
  DevBuf hamming, hist_seg[2], hist_map[2], plan, header, turns, total;
  int cur = 0, n_hist = 0, cap_B = 0;
  int turn_cap = 0;
  PinnedBuf pin;                  // pinned staging: plan in, header + total + turn prefix out
};

static const int DG_POST_PREFIX = 16384;   // turns copied back together with the header (one D2H in the common case)

extern "C" int dg_post_create(int frames, int local_speakers, int max_speakers, int num_windows, const double* hamming_host,
                              double tau, int device, dg_post** out) {
  if (!out || !hamming_host || frames < 1 || frames > 1023 || local_speakers < 1 || max_speakers < 1 || max_speakers > 64 ||
      num_windows < 1 || num_windows > 256) {
    set_error("dg_post_create: need 1 <= frames <= 1023, 1 <= max_speakers <= 64, 1 <= num_windows <= 256");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_post> h(new dg_post());
  h->device = device; h->F = frames; h->K = local_speakers; h->M = max_speakers; h->nw = num_windows; h->tau = tau;
  if (h->hamming.ensure((size_t)frames * 8) || h->total.ensure(16)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, (size_t)frames * 8, cudaMemcpyHostToDevice));
  const size_t hs = (size_t)std::max(1, num_windows - 1);
  for (int i = 0; i < 2; i++)
    if (h->hist_seg[i].ensure(hs * frames * local_speakers * 4) || h->hist_map[i].ensure(hs * local_speakers * 4)) return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_post_reset(dg_post* h) {
  if (!h) return DG_EINVAL;
  h->n_hist = 0;
  return DG_OK;
}

extern "C" int dg_post_destroy(dg_post* h) {
  delete h;
  return DG_OK;
}

static int post_ensure(dg_post* h, int B) {
  if (B <= h->cap_B) return 0;
  const int stride = 4 + h->nw;
  // worst case: every second frame of every speaker starts a turn
  h->turn_cap = B * h->M * ((h->F + 1) / 2);
  if (h->plan.ensure((size_t)B * stride * 4) || h->header.ensure((size_t)B * 16 + 16) ||
      h->turns.ensure((size_t)h->turn_cap * 4))
    return DG_ECUDA;
  if (h->pin.ensure((size_t)B * stride * 4 + (size_t)B * 16 + 16 + (size_t)DG_POST_PREFIX * 4)) return DG_ECUDA;
  h->cap_B = B;
  return 0;
}

// enqueues plan upload, aggregation + binarisation + run-length kernel, history update and the D2H of the results on `st`
static int post_enqueue(dg_post* h, const float* seg_dev, const int32_t* map_dev, int B, const int32_t* plan_host,
                        cudaStream_t st) {
  int rc;
  if ((rc = post_ensure(h, B))) return rc;
  const int stride = 4 + h->nw;
  unsigned char* pin = h->pin.as<unsigned char>();
  const size_t plan_bytes = (size_t)B * stride * 4;
  memcpy(pin, plan_host, plan_bytes);
  DG_CUDA(cudaMemcpyAsync(h->plan.p, pin, plan_bytes, cudaMemcpyHostToDevice, st));
  DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
  if ((rc = launch_post(seg_dev, map_dev, h->hist_seg[h->cur].as<float>(), h->hist_map[h->cur].as<int32_t>(), h->n_hist, B,
                        h->F, h->K, h->M, h->nw, h->plan.as<int32_t>(), stride, h->hamming.as<double>(), h->tau,
                        h->header.as<int32_t>(), h->turns.as<uint32_t>(), h->turn_cap, h->total.as<unsigned int>(), st)))
    return rc;
  const int keep = std::min(h->nw - 1, h->n_hist + B);
  if (keep > 0) {
    if ((rc = launch_post_history(seg_dev, map_dev, h->hist_seg[h->cur].as<float>(), h->hist_map[h->cur].as<int32_t>(),
                                  h->n_hist, B, h->F, h->K, keep, h->hist_seg[h->cur ^ 1].as<float>(),
                                  h->hist_map[h->cur ^ 1].as<int32_t>(), st)))
      return rc;
    h->cur ^= 1;
  }
  h->n_hist = keep;
  unsigned char* out = pin + plan_bytes;
  DG_CUDA(cudaMemcpyAsync(out, h->header.p, (size_t)B * 16, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(out + (size_t)B * 16, h->total.p, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(out + (size_t)B * 16 + 16, h->turns.p, (size_t)std::min(DG_POST_PREFIX, h->turn_cap) * 4,
                          cudaMemcpyDeviceToHost, st));
  return 0;
}

// after `st` has been synchronised: hands the results to the caller
static int post_finish(dg_post* h, int B, int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                       cudaStream_t st) {
  const int stride = 4 + h->nw;
  unsigned char* out = h->pin.as<unsigned char>() + (size_t)B * stride * 4;
  unsigned int total = 0;
  memcpy(&total, out + (size_t)B * 16, 4);
  if (n_turns) *n_turns = (int)total;
  memcpy(header_host, out, (size_t)B * 16);
  if ((int)total > turn_cap_host) {
    set_error("dg_post_step: turn buffer too small (" + std::to_string(total) + " turns)");
    return DG_EINVAL;
  }
  const unsigned int pre = std::min<unsigned int>(total, (unsigned int)DG_POST_PREFIX);
  memcpy(turns_host, out + (size_t)B * 16 + 16, (size_t)pre * 4);
  if (total > pre) {
    DG_CUDA(cudaMemcpyAsync(turns_host + pre, h->turns.as<uint32_t>() + pre, (size_t)(total - pre) * 4,
                            cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
  }
  return DG_OK;
}

extern "C" int dg_post_step(dg_post* h, const float* seg_dev, const int32_t* map_dev, int B, const int32_t* plan_host,
                            int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  if (!h || !seg_dev || !map_dev || !plan_host || !header_host || !turns_host || B < 1) {
    set_error("dg_post_step: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = post_enqueue(h, seg_dev, map_dev, B, plan_host, st))) return rc;
  DG_CUDA(cudaStreamSynchronize(st));
  return post_finish(h, B, header_host, turns_host, turn_cap_host, n_turns, st);
}

// ============================================================================= hyper-parameter sweep
// T independent clustering + post-path states over ONE set of network outputs (seg, emb of a whole file): the reference tunes
// tau_active, rho_update and delta_new by re-running its whole pipeline per trial (Optimizer.objective -> Benchmark), although
// none of the three reaches the networks.  Clustering: one CTA per state (cluster.cu); post-path: one CTA per (chunk, state)
// over all chunks at once, without history (post.cu).
struct dg_sweep {
  int device = 0, M = 0, D = 0, F = 0, K = 0, nw = 1;
  DevBuf hamming, in, centers, active, init, prep, prep_d, maps, header, turns, total;
  DevBuf score_in, hoff, hseg, comp;   // dg_sweep_score: chunk times and reference, hypothesis segments, components
  PinnedBuf pin;                  // params, taus and plan in; error flags, header, total and a turn prefix out
};

extern "C" int dg_sweep_create(int max_speakers, int dim, int frames, int local_speakers, int num_windows,
                               const double* hamming_host, int device, dg_sweep** out) {
  if (!out || !hamming_host || max_speakers < 1 || max_speakers > 32 || dim < 1 || local_speakers < 1 || local_speakers > 8 ||
      local_speakers > max_speakers || frames < 1 || frames > 1023 || num_windows < 1 || num_windows > 256) {
    set_error("dg_sweep_create: need 1 <= max_speakers <= 32, dim >= 1, 1 <= local_speakers <= min(8, max_speakers), "
              "1 <= frames <= 1023, 1 <= num_windows <= 256");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_sweep> h(new dg_sweep());
  h->device = device; h->M = max_speakers; h->D = dim; h->F = frames; h->K = local_speakers; h->nw = num_windows;
  if (h->hamming.ensure((size_t)frames * 8) || h->total.ensure(16)) return DG_ECUDA;
  DG_CUDA(cudaMemcpy(h->hamming.p, hamming_host, (size_t)frames * 8, cudaMemcpyHostToDevice));
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_sweep_destroy(dg_sweep* h) {
  delete h;
  return DG_OK;
}

// the argument checks dg_sweep_run and dg_sweep_score share (before any launch)
static int sweep_check(const char* who, dg_sweep* h, const float* seg_dev, const float* emb_dev, int N,
                       const double* params_host, int T, const int32_t* plan_host) {
  if (!h || !seg_dev || !emb_dev || !params_host || !plan_host || N < 1 || T < 1 || T > 65535) {
    set_error(std::string(who) + ": bad arguments (need N >= 1, 1 <= T <= 65535, non-null buffers)");
    return DG_EINVAL;
  }
  for (int i = 0; i < 3 * T; i++)
    if (!std::isfinite(params_host[i])) {
      set_error(std::string(who) + ": trial " + std::to_string(i / 3) + " has a parameter that is not finite");
      return DG_EINVAL;
    }
  return DG_OK;
}

// pinned output layout of sweep_cluster_post: error flags [T][2], header [T][N][4], total (16 bytes), a prefix of the turns
static size_t sweep_out_bytes(int T, int N) { return (size_t)T * 8 + (size_t)T * N * 16 + 16 + (size_t)DG_POST_PREFIX * 4; }

// Clustering + post-path of T trials over the N chunks: header [T][N][4] and turns stay on the device (h->header, h->turns),
// the turn count comes back in *total.  with_header: the header and a prefix of the turns travel to the pinned buffer in the
// same copy as the count (sweep_out_bytes layout).  Synchronises `st`.
static int sweep_cluster_post(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host,
                              int T, const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, bool with_header,
                              cudaStream_t st, unsigned int* total_out) {
  const int stride = 4 + h->nw, M = h->M, D = h->D, K = h->K, F = h->F;
  // host -> device: params [T][3], taus [T], plan [N][stride], one copy
  const size_t params_b = (size_t)T * 24, taus_b = (size_t)T * 8, plan_b = (size_t)N * stride * 4;
  const size_t in_b = params_b + taus_b + plan_b;
  const size_t init_b = (size_t)T * 8, header_b = (size_t)T * N * 16;
  const size_t out_b = sweep_out_bytes(T, N);
  // the device turn buffer starts at a guess and grows to the true count (the kernel counts every turn, writes those that fit)
  const size_t turn_guess = std::max<size_t>((size_t)T * N * 8, (size_t)DG_POST_PREFIX);
  if (h->in.ensure(in_b) || h->centers.ensure((size_t)T * M * D * 8) || h->active.ensure((size_t)T * 32 * 4) ||
      h->init.ensure(init_b) || h->prep.ensure(cluster_prep_floats(N, K) * 4 + 16) ||
      h->prep_d.ensure(cluster_prep_doubles(N, K) * 8 + 16) || (!maps_dev && h->maps.ensure((size_t)T * N * K * 4)) ||
      h->header.ensure(header_b) || h->turns.ensure(turn_guess * 4) || h->pin.ensure(std::max(in_b, out_b)))
    return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  double* p_taus = reinterpret_cast<double*>(pin + params_b);
  memcpy(pin, params_host, params_b);
  for (int t = 0; t < T; t++) p_taus[t] = params_host[3 * t];
  memcpy(pin + params_b + taus_b, plan_host, plan_b);
  unsigned char* din = h->in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const double* d_params = reinterpret_cast<const double*>(din);
  const double* d_taus = reinterpret_cast<const double*>(din + params_b);
  const int32_t* d_plan = reinterpret_cast<const int32_t*>(din + params_b + taus_b);
  int32_t* maps = maps_dev ? maps_dev : h->maps.as<int32_t>();
  // every state starts empty (reference: a new OnlineSpeakerClustering per trial)
  DG_CUDA(cudaMemsetAsync(h->centers.p, 0, (size_t)T * M * D * 8, st));
  DG_CUDA(cudaMemsetAsync(h->active.p, 0, (size_t)T * 32 * 4, st));
  DG_CUDA(cudaMemsetAsync(h->init.p, 0, init_b, st));
  ClusterParams p{};
  p.M = M;
  p.D = D;
  p.metric = 0;
  int rc;
  if ((rc = launch_cluster_sweep(p, d_params, T, seg_dev, emb_dev, N, F, K, h->centers.as<double>(), h->active.as<int>(),
                                 h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), maps, st)))
    return rc;
  if (centers_dev)
    DG_CUDA(cudaMemcpyAsync(centers_dev, h->centers.p, (size_t)T * M * D * 8, cudaMemcpyDeviceToDevice, st));
  unsigned int total = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    const int cap = (int)std::min<size_t>(h->turns.bytes / 4, (size_t)INT32_MAX);
    DG_CUDA(cudaMemsetAsync(h->total.p, 0, 4, st));
    if ((rc = launch_post(seg_dev, maps, nullptr, nullptr, 0, N, F, K, M, h->nw, d_plan, stride, h->hamming.as<double>(), 0.0,
                          h->header.as<int32_t>(), h->turns.as<uint32_t>(), cap, h->total.as<unsigned int>(), st, d_taus, T)))
      return rc;
    DG_CUDA(cudaMemcpyAsync(pin, h->init.p, init_b, cudaMemcpyDeviceToHost, st));
    if (with_header) DG_CUDA(cudaMemcpyAsync(pin + init_b, h->header.p, header_b, cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaMemcpyAsync(pin + init_b + header_b, h->total.p, 4, cudaMemcpyDeviceToHost, st));
    if (with_header)
      DG_CUDA(cudaMemcpyAsync(pin + init_b + header_b + 16, h->turns.p, (size_t)std::min(DG_POST_PREFIX, cap) * 4,
                              cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
    memcpy(&total, pin + init_b + header_b, 4);
    if (total <= (unsigned int)cap) break;
    // more turns than the device buffer holds: grow it to the count and binarise again (the maps are unchanged)
    if (h->turns.ensure((size_t)total * 4)) return DG_ECUDA;
  }
  const int32_t* flags = reinterpret_cast<const int32_t*>(pin);
  for (int t = 0; t < T; t++)
    if (flags[2 * t + 1]) {
      set_error("Cannot update unknown centers");   // reference clustering.py:98 (AssertionError)
      return DG_EINVAL;
    }
  *total_out = total;
  return DG_OK;
}

extern "C" int dg_sweep_run(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host, int T,
                            const int32_t* plan_host, int32_t* maps_dev, double* centers_dev, int32_t* header_host,
                            uint32_t* turns_host, int turn_cap_host, int* n_turns, void* stream) {
  if (!header_host || !turns_host) {
    set_error("dg_sweep_run: bad arguments (need N >= 1, 1 <= T <= 65535, non-null buffers)");
    return DG_EINVAL;
  }
  int rc;
  if ((rc = sweep_check("dg_sweep_run", h, seg_dev, emb_dev, N, params_host, T, plan_host))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, params_host, T, plan_host, maps_dev, centers_dev, true, st, &total)))
    return rc;
  const unsigned char* pin = h->pin.as<unsigned char>();
  const size_t init_b = (size_t)T * 8, header_b = (size_t)T * N * 16;
  if (n_turns) *n_turns = (int)total;
  memcpy(header_host, pin + init_b, header_b);
  if ((long long)total > (long long)turn_cap_host) {
    set_error("dg_sweep_run: turn buffer too small (" + std::to_string(total) + " turns)");
    return DG_EINVAL;
  }
  const unsigned int pre = std::min<unsigned int>(total, (unsigned int)DG_POST_PREFIX);
  memcpy(turns_host, pin + init_b + header_b + 16, (size_t)pre * 4);
  if (total > pre) {     // a second copy for what did not travel with the header
    DG_CUDA(cudaMemcpyAsync(turns_host + pre, h->turns.as<uint32_t>() + pre, (size_t)(total - pre) * 4,
                            cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
  }
  return DG_OK;
}

// the reference rows: finite, start < end, labels in [0, R), each label's rows in time order without overlap
static int sweep_check_reference(const double* ref_host, const int32_t* ref_label_host, int S, int R) {
  if (R < 0 || R > 32 || S < 0 || (S > 0 && (!ref_host || !ref_label_host))) {
    set_error("dg_sweep_score: need 0 <= reference labels <= 32, rows >= 0, non-null reference arrays");
    return DG_EINVAL;
  }
  double last[32];
  for (int r = 0; r < 32; r++) last[r] = -INFINITY;
  for (int i = 0; i < S; i++) {
    const double a = ref_host[2 * i], b = ref_host[2 * i + 1];
    const int r = ref_label_host[i];
    if (r < 0 || r >= R) {
      set_error("dg_sweep_score: reference row " + std::to_string(i) + " has a label outside [0, R)");
      return DG_EINVAL;
    }
    if (!std::isfinite(a) || !std::isfinite(b) || !(a < b)) {
      set_error("dg_sweep_score: reference row " + std::to_string(i) + " is not finite, empty or reversed");
      return DG_EINVAL;
    }
    if (a < last[r]) {
      set_error("dg_sweep_score: reference row " + std::to_string(i) + " is out of order or overlaps an earlier row of its label");
      return DG_EINVAL;
    }
    last[r] = b;
  }
  return DG_OK;
}

extern "C" int dg_sweep_score(dg_sweep* h, const float* seg_dev, const float* emb_dev, int N, const double* params_host,
                              int T, const int32_t* plan_host, const double* out_start_host, const double* out_res_host,
                              double shift, double collar, const double* ref_host, const int32_t* ref_label_host, int S,
                              int R, double* components_host, int32_t* hyp_offsets_dev, double* hyp_segments_dev,
                              int hyp_cap, void* stream) {
  int rc;
  if ((rc = sweep_check("dg_sweep_score", h, seg_dev, emb_dev, N, params_host, T, plan_host))) return rc;
  if (!out_start_host || !out_res_host || !components_host || hyp_cap < 0 || !std::isfinite(shift) ||
      !std::isfinite(collar) || collar < 0) {
    set_error("dg_sweep_score: bad arguments (need chunk times, a components buffer, finite shift, finite collar >= 0, "
              "hyp_cap >= 0)");
    return DG_EINVAL;
  }
  for (int c = 0; c < N; c++)
    if (!std::isfinite(out_start_host[c]) || !std::isfinite(out_res_host[c])) {
      set_error("dg_sweep_score: chunk " + std::to_string(c) + " has an output time that is not finite");
      return DG_EINVAL;
    }
  if ((rc = sweep_check_reference(ref_host, ref_label_host, S, R))) return rc;
  DG_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int total = 0;
  if ((rc = sweep_cluster_post(h, seg_dev, emb_dev, N, params_host, T, plan_host, nullptr, nullptr, false, st, &total)))
    return rc;
  const int M = h->M, TM = T * M;
  // host -> device, one copy: out_start [N], out_res [N], reference segments [S][2] grouped by label, label offsets [R + 1]
  const size_t times_b = (size_t)N * 16, rseg_b = (size_t)S * 16, roff_b = (size_t)(R + 1) * 4;
  const size_t in_b = times_b + rseg_b + roff_b, comp_b = (size_t)T * 40;
  if (h->score_in.ensure(in_b) || h->hoff.ensure((size_t)(TM + 1) * 4) || h->hseg.ensure((size_t)std::max(total, 1u) * 16) ||
      h->comp.ensure(comp_b) || h->pin.ensure(std::max(in_b, comp_b + 16)))
    return DG_ECUDA;
  unsigned char* pin = h->pin.as<unsigned char>();
  memcpy(pin, out_start_host, (size_t)N * 8);
  memcpy(pin + (size_t)N * 8, out_res_host, (size_t)N * 8);
  double* rseg = reinterpret_cast<double*>(pin + times_b);
  int32_t* roff = reinterpret_cast<int32_t*>(pin + times_b + rseg_b);
  for (int r = 0; r <= R; r++) roff[r] = 0;
  for (int i = 0; i < S; i++) roff[ref_label_host[i] + 1]++;
  for (int r = 0; r < R; r++) roff[r + 1] += roff[r];
  int fill[32];
  for (int r = 0; r < R; r++) fill[r] = roff[r];
  for (int i = 0; i < S; i++) {     // stable: each label keeps its rows' order
    const int o = fill[ref_label_host[i]]++;
    rseg[2 * o] = ref_host[2 * i];
    rseg[2 * o + 1] = ref_host[2 * i + 1];
  }
  unsigned char* din = h->score_in.as<unsigned char>();
  DG_CUDA(cudaMemcpyAsync(din, pin, in_b, cudaMemcpyHostToDevice, st));
  const double* d_start = reinterpret_cast<const double*>(din);
  const double* d_res = d_start + N;
  const double* d_rseg = reinterpret_cast<const double*>(din + times_b);
  const int* d_roff = reinterpret_cast<const int*>(din + times_b + rseg_b);
  int* hoff = h->hoff.as<int>();
  if ((rc = launch_der_hyp_count(h->header.as<int32_t>(), h->turns.as<uint32_t>(), T, N, M, d_start, d_res, shift, collar,
                                 hoff, st)) ||
      (rc = launch_der_hyp_write(h->header.as<int32_t>(), h->turns.as<uint32_t>(), T, N, M, d_start, d_res, shift, collar,
                                 hoff, h->hseg.as<double>(), hyp_segments_dev, hyp_cap, st)) ||
      (rc = launch_der_score(hoff, h->hseg.as<double>(), T, M, d_roff, d_rseg, R, h->comp.as<double>(), st)))
    return rc;
  if (hyp_offsets_dev) DG_CUDA(cudaMemcpyAsync(hyp_offsets_dev, hoff, (size_t)(TM + 1) * 4, cudaMemcpyDeviceToDevice, st));
  DG_CUDA(cudaMemcpyAsync(pin, h->comp.p, comp_b, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaMemcpyAsync(pin + comp_b, hoff + TM, 4, cudaMemcpyDeviceToHost, st));
  DG_CUDA(cudaStreamSynchronize(st));
  memcpy(components_host, pin, comp_b);
  int n_seg = 0;
  memcpy(&n_seg, pin + comp_b, 4);
  if (hyp_segments_dev && n_seg > hyp_cap) {
    set_error("dg_sweep_score: hypothesis segment buffer too small (" + std::to_string(n_seg) + " segments)");
    return DG_EINVAL;
  }
  return DG_OK;
}

// worker threads of the host gather, created at the first dg_pipeline_call_host: all cores but two, at most 24
static GatherPool& gather_pool(dg_pipeline* h) {
  if (!h->gather) h->gather.reset(new GatherPool(std::max(1, std::min((int)std::thread::hardware_concurrency() - 2, 24))));
  return *h->gather;
}

// ---- the whole body of SpeakerDiarization.__call__ (reference diarization.py:172-232) in one call: B separate host windows
//      (as rearrange_audio_stream emits them) are gathered into pinned staging by worker threads while earlier rows are
//      already on their way to the device, then fused step + post-path, one D2H of the turn list.
static int upload_rows(dg_pipeline* h, const float* const* rows, int B, int S, float* pin, float* dst_dev, cudaStream_t st) {
  const int R = 4;                                    // rows per work item (1.3 MB at S = 80000)
  const int items = (B + R - 1) / R;
  GatherPool& pool = gather_pool(h);
  std::vector<std::atomic<int>> done(items);
  for (auto& d : done) d.store(0, std::memory_order_relaxed);
  std::atomic<int> next{0};
  pool.start([&]() {
    for (;;) {
      const int it = next.fetch_add(1, std::memory_order_relaxed);
      if (it >= items) return;
      const int r0 = it * R, r1 = std::min(B, r0 + R);
      for (int r = r0; r < r1; r++) memcpy(pin + (size_t)r * S, rows[r], (size_t)S * 4);
      done[it].store(1, std::memory_order_release);
    }
  });
  // the calling thread forwards finished items, in order, in runs of up to 8 (~10 MB per copy)
  cudaError_t err = cudaSuccess;
  int sent = 0;
  while (sent < items) {
    int upto = sent;
    while (upto < items && upto - sent < 8 && done[upto].load(std::memory_order_acquire)) upto++;
    if (upto == sent) {
      std::this_thread::yield();
      continue;
    }
    const int r0 = sent * R, r1 = std::min(B, upto * R);
    if (err == cudaSuccess)
      err = cudaMemcpyAsync(dst_dev + (size_t)r0 * S, pin + (size_t)r0 * S, (size_t)(r1 - r0) * S * 4, cudaMemcpyHostToDevice, st);
    sent = upto;
  }
  pool.wait();          // (`next` and `done` live on this frame)
  DG_CUDA(err);
  return 0;
}

// Windows that are consecutive hops of ONE stream -- what the reference's rearrange_audio_stream emits (operators.py:44-100) --
// share S - hop samples with their neighbour.  The workers compare every window with its predecessor (memcmp of the shared
// samples, exact) and pack the `hop` new samples of each into the pinned stream image; the caller then uploads
// S + (B - 1) hop samples instead of B S and forms the windows on the device.  Returns 1 if windows [r0, r0 + nb) continue the
// stream (pin_stream[0 .. S + (r0 + nb - 1) hop) is then valid), 0 if some window does not (the caller falls back to the
// full gather for this and the following sub-batches).
static int pack_stream_rows(dg_pipeline* h, const float* const* rows, int r0, int nb, int S, int hop, float* pin_stream) {
  GatherPool& pool = gather_pool(h);
  std::atomic<int> next{r0}, bad{0};
  pool.start([&]() {
    for (;;) {
      const int r = next.fetch_add(1, std::memory_order_relaxed);
      if (r >= r0 + nb || bad.load(std::memory_order_relaxed)) return;
      if (r == 0) {
        memcpy(pin_stream, rows[0], (size_t)S * 4);
      } else if (memcmp(rows[r - 1] + hop, rows[r], (size_t)(S - hop) * 4) != 0) {
        bad.store(1, std::memory_order_relaxed);
      } else {
        memcpy(pin_stream + (size_t)S + (size_t)(r - 1) * hop, rows[r] + (S - hop), (size_t)hop * 4);
      }
    }
  });
  pool.wait();
  return bad.load() ? 0 : 1;
}

static bool post_fits(const dg_pipeline* h, const dg_post* post, const StepShape& sh) {
  return sh.F == post->F && sh.K == post->K && h->clu->p.M == post->M && post->device == h->seg->device;
}

// end of dg_pipeline_call_host / _call_stream, with the batch's scores and maps in segd / mapd (ordered on h->st): post-path,
// optional downloads, one synchronise (time stamp in *synced, if given), turn list
static int call_finish(dg_pipeline* h, dg_post* post, const StepShape& sh, const int32_t* plan_host, int32_t* header_host,
                       uint32_t* turns_host, int turn_cap_host, int* n_turns, float* seg_host, int32_t* map_host,
                       std::chrono::steady_clock::time_point* synced) {
  int rc;
  const StepOut dev = {h->segd.as<float>(), nullptr, h->mapd.as<int32_t>(), nullptr};
  if ((rc = post_enqueue(post, dev.seg, dev.map, sh.B, plan_host, h->st))) return rc;
  if ((rc = copy_out(h, h->st, nullptr, sh, dev, {seg_host, nullptr, map_host, nullptr}, cudaMemcpyDeviceToHost))) return rc;
  DG_CUDA(cudaStreamSynchronize(h->st));
  if (synced) *synced = std::chrono::steady_clock::now();
  return post_finish(post, sh.B, header_host, turns_host, turn_cap_host, n_turns, h->st);
}

extern "C" int dg_pipeline_call_host(dg_pipeline* h, dg_post* post, const float* const* rows_host, int B, int S,
                                     const int32_t* plan_host, int32_t* header_host, uint32_t* turns_host, int turn_cap_host,
                                     int* n_turns, float* seg_host, int32_t* map_host) {
  if (!h || !post || !rows_host || !plan_host || !header_host || !turns_host || B < 1) {
    set_error("dg_pipeline_call_host: bad arguments");
    return DG_EINVAL;
  }
  int rc;
  StepShape sh = {B};
  if ((rc = dg_seg_dims(h->seg, S, &sh.F, &sh.K))) return rc;
  if (!post_fits(h, post, sh)) {
    set_error("dg_pipeline_call_host: post handle was created for other dimensions");
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error("dg_pipeline_call_host: submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  // DG_CALL_TIMING=1: host wall-clock phases of the call on stderr (diagnostic)
  static const bool call_timing = getenv("DG_CALL_TIMING") && getenv("DG_CALL_TIMING")[0] == '1';
  const auto tc0 = std::chrono::steady_clock::now();
  static thread_local CallDiag diag;
  if (call_timing) {
    diag.create();
    cudaEventRecord(diag.t0, h->s_h2d);
    g_diag = &diag;
  }
  if (h->segd.ensure(sh.seg_bytes()) || h->mapd.ensure(sh.map_bytes())) return DG_ECUDA;
  if (h->pin_wav.ensure((size_t)B * S * 4)) return DG_ECUDA;
  // The batch runs as up to three sub-batches through the pipelined machinery (dg_pipeline_submit_host): the upload of
  // sub-batch j+1 and its front end overlap the recurrence of sub-batch j; clustering stays in chunk order on its one stream,
  // so the result is exactly that of one step over the whole batch.  From 64 windows on: two halves; from 192 windows on:
  // three parts -- a short first one so that the device starts early and a short last one, because its dependent chain
  // (1172 recurrence steps + its share of the clustering) is what the caller waits for at the end
  int plan[DG_MAX_INFLIGHT] = {B, 0, 0}, ns = 1;
  if (B >= 192) {
    ns = 3;
    plan[0] = (B * 5 / 16 + 7) / 8 * 8;
    plan[2] = (B * 4 / 16 + 7) / 8 * 8;
    plan[1] = B - plan[0] - plan[2];
  } else if (B >= 64) {
    ns = 2;
    plan[0] = (B / 2 + 7) / 8 * 8;
    plan[1] = B - plan[0];
  }
  // consecutive windows of one stream (hop known from dg_pipeline_set_hop): verified on the host, uploaded once (see
  // pack_stream_rows)
  const int hop = h->hop;
  bool as_stream = hop > 0 && hop < S && hop % 4 == 0 && S % 4 == 0 && B >= 2;
  const size_t stream_len = (size_t)S + (size_t)(B - 1) * (hop > 0 ? hop : 0);
  if (as_stream && h->call_stream.ensure((stream_len + 64) * 4)) return DG_ECUDA;
  float* pin = h->pin_wav.as<float>();
  h->call_h2d_bytes = 0;
  for (int j = 0, r0 = 0; j < ns; r0 += plan[j], j++) {
    const int nb = plan[j];
    const int slot = (int)(h->next_step % 3);
    if (h->slot_wav[slot].ensure((size_t)nb * S * 4)) return DG_ECUDA;
    DG_CUDA(cudaStreamWaitEvent(h->s_h2d, h->e_slot_done[slot], 0));
    if (as_stream && !pack_stream_rows(h, rows_host, r0, nb, S, hop, pin)) as_stream = false;
    int stream_hop = 0;
    if (as_stream) {
      // the samples this sub-batch adds to the device image of the stream, then its windows from that image
      const size_t lo = r0 == 0 ? 0 : (size_t)S + (size_t)(r0 - 1) * hop, hi = (size_t)S + (size_t)(r0 + nb - 1) * hop;
      DG_CUDA(cudaMemcpyAsync(h->call_stream.as<float>() + lo, pin + lo, (hi - lo) * 4, cudaMemcpyHostToDevice, h->s_h2d));
      h->call_h2d_bytes += (long long)(hi - lo) * 4;
      const long long cap = (long long)((stream_len + 3) / 4 * 4 + 4);     // linear image: the ring index never wraps
      if ((rc = launch_expand_windows(h->call_stream.as<float>(), (long long)r0 * hop, (int)cap, hop, S, nb,
                                      h->slot_wav[slot].as<float>(), h->s_h2d)))
        return rc;
      stream_hop = hop;
    } else {
      // (after a failed stream check the pinned buffer is reused as the [B, S] staging: earlier sub-batches are already on the device)
      if (h->call_h2d_bytes) DG_CUDA(cudaStreamSynchronize(h->s_h2d));
      if ((rc = upload_rows(h, rows_host + r0, nb, S, pin + (size_t)r0 * S, h->slot_wav[slot].as<float>(), h->s_h2d))) return rc;
      h->call_h2d_bytes += (long long)nb * S * 4;
    }
    DG_CUDA(cudaEventRecord(h->e_h2d[slot], h->s_h2d));
    if (g_diag) g_diag->j = j;
    DG_DIAG(up, h->s_h2d);
    if ((rc = pipeline_submit(h, h->slot_wav[slot].as<float>(), S, {nb, sh.F, sh.K}, h->e_h2d[slot], stream_hop))) return rc;
  }
  for (int j = 0, r0 = 0; j < ns; r0 += plan[j], j++)     // collect the sub-batches' scores / maps, in order
    if ((rc = dg_pipeline_collect_copy(h, h->segd.as<float>() + (size_t)r0 * sh.F * sh.K, nullptr,
                                       h->mapd.as<int32_t>() + (size_t)r0 * sh.K, h->st)))
      return rc;
  const auto tc1 = std::chrono::steady_clock::now();
  auto tc2 = tc1;
  rc = call_finish(h, post, sh, plan_host, header_host, turns_host, turn_cap_host, n_turns, seg_host, map_host, &tc2);
  g_diag = nullptr;
  if (call_timing) {
    static int shown = 0;
    if (rc == 0 && shown++ % 4 == 3) {
      for (int j = 0; j < ns; j++) {
        float t[6] = {0, 0, 0, 0, 0, 0};
        cudaEvent_t ev[6] = {diag.up[j], diag.prep[j], diag.trunk[j], diag.seg[j], diag.emb[j], diag.clu[j]};
        for (int q = 0; q < 6; q++) cudaEventElapsedTime(&t[q], diag.t0, ev[q]);
        fprintf(stderr, "  sub-batch %d (%d windows), ms after entry: uploaded %.2f | front end %.2f | embedding trunk %.2f | segmentation + "
                        "OSP %.2f | embeddings %.2f | clustered %.2f\n", j, plan[j], t[0], t[1], t[2], t[3], t[4], t[5]);
      }
    }
    static double acc[3] = {0, 0, 0};
    static int calls = 0;
    const auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
      return std::chrono::duration<double, std::milli>(b - a).count(); };
    acc[0] += ms(tc0, tc1);
    acc[1] += ms(tc1, tc2);
    acc[2] += ms(tc2, std::chrono::steady_clock::now());
    if (++calls % 4 == 0) {
      fprintf(stderr, "dg_pipeline_call_host (B=%d, %d sub-batches): gather + upload + enqueue %.2f ms | wait for the device %.2f ms | "
                      "turn list %.2f ms (mean of 4 calls)\n", B, ns, acc[0] / 4, acc[1] / 4, acc[2] / 4);
      acc[0] = acc[1] = acc[2] = 0;
    }
  }
  return rc;
}

extern "C" int64_t dg_pipeline_last_call_h2d_bytes(const dg_pipeline* h) { return h ? (int64_t)h->call_h2d_bytes : 0; }

// ---- shared-identity mode (SURVEY.md 8(e), BASELINE config 5) without leaving the pipelined flow.  After dg_pipeline_submit*:
//   dg_pipeline_identity_export  enqueues the export of this rank's centroid changes behind the clustering of every submitted
//                                step (clustering stream) and makes `stream` wait for it -> the caller all-gathers the records
//   dg_pipeline_identity_merge   makes the clustering stream wait for `stream` (the all-gather), merges all ranks' records and
//                                relabels the speaker maps of the steps clustered since the previous merge (still on the device)
// The clustering of the NEXT submitted step is ordered behind the merge, exactly as in the one-step-at-a-time protocol; only
// the networks of the next steps overlap the exchange.  Call the pair once after every submit, before collecting that step.
extern "C" int dg_pipeline_identity_export(dg_pipeline* h, double* record_dev, void* stream) {
  if (!h || !record_dev) {
    set_error("dg_pipeline_identity_export: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  if (!h->e_ident && (h->e_ident.create() || h->e_ident_in.create())) return DG_ECUDA;
  int rc;
  if ((rc = dg_cluster_export_delta(h->clu, record_dev, h->s_clu))) return rc;
  DG_CUDA(cudaEventRecord(h->e_ident, h->s_clu));
  DG_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->e_ident, 0));
  return DG_OK;
}

extern "C" int dg_pipeline_identity_merge(dg_pipeline* h, const double* records_dev, int world, int rank, void* stream) {
  if (!h || !records_dev || world < 1 || rank < 0 || rank >= world || !h->e_ident) {
    set_error("dg_pipeline_identity_merge: bad arguments (or no export before it)");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  DG_CUDA(cudaEventRecord(h->e_ident_in, (cudaStream_t)stream));
  DG_CUDA(cudaStreamWaitEvent(h->s_clu, h->e_ident_in, 0));
  int rc;
  long long first = h->ident_merged_upto;
  if (first < h->next_step - DG_MAX_INFLIGHT) first = h->next_step - DG_MAX_INFLIGHT;
  bool merged = false;
  for (long long step = first; step < h->next_step; step++) {
    const int slot = (int)(step % 3);
    int32_t* maps = h->slot_map[slot].as<int32_t>();
    const int n = h->slot_shape[slot].B * h->slot_shape[slot].K;
    if (!merged) {
      if ((rc = dg_cluster_merge(h->clu, records_dev, world, rank, maps, n, h->s_clu))) return rc;
      merged = true;
    } else if ((rc = launch_relabel_maps(maps, n, h->clu->relabel.as<int32_t>(), h->s_clu))) {
      return rc;
    }
    DG_CUDA(cudaEventRecord(h->e_slot_done[slot], h->s_clu));      // collect must see the relabelled maps
  }
  if (!merged && (rc = dg_cluster_merge(h->clu, records_dev, world, rank, nullptr, 0, h->s_clu))) return rc;
  h->ident_merged_upto = h->next_step;
  return DG_OK;
}

// pipelined step whose batch is the next B windows of a device-side stream (no window upload at all; the sinc layer takes
// its stream form without the overlap check: the windows overlap by construction)
extern "C" int dg_pipeline_submit_stream(dg_pipeline* h, dg_stream* s, int B) {
  if (!h || !s || B < 1) {
    set_error("dg_pipeline_submit_stream: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding >= DG_MAX_INFLIGHT) {
    set_error("dg_pipeline_submit_stream: three steps are already outstanding; collect one first");
    return DG_EINVAL;
  }
  if (s->device != h->seg->device) {
    set_error("dg_pipeline_submit_stream: stream and pipeline live on different devices");
    return DG_EINVAL;
  }
  int rc, F = 0, K = 0;
  const int S = stream_window_len(s);
  if ((rc = dg_seg_dims(h->seg, S, &F, &K))) return rc;
  DG_CUDA(cudaSetDevice(h->seg->device));
  const int slot = (int)(h->next_step % 3);
  if (h->slot_wav[slot].ensure((size_t)B * S * 4)) return DG_ECUDA;
  DG_CUDA(cudaStreamWaitEvent(h->s_h2d, h->e_slot_done[slot], 0));
  if ((rc = stream_expand(s, B, h->slot_wav[slot].as<float>(), h->s_h2d))) return rc;
  DG_CUDA(cudaEventRecord(h->e_h2d[slot], h->s_h2d));
  // resampled windows differ from exact hops of one stream at their edges: no stream-form claim for them
  return pipeline_submit(h, h->slot_wav[slot].as<float>(), S, {B, F, K}, h->e_h2d[slot], s->rs ? 0 : s->hop);
}

// SpeakerDiarization.__call__ for the next B windows of a device-side stream: fused step + post-path, synchronous
extern "C" int dg_pipeline_call_stream(dg_pipeline* h, dg_post* post, dg_stream* s, int B, const int32_t* plan_host,
                                       int32_t* header_host, uint32_t* turns_host, int turn_cap_host, int* n_turns,
                                       float* seg_host, int32_t* map_host) {
  if (!h || !post || !s || !plan_host || !header_host || !turns_host || B < 1) {
    set_error("dg_pipeline_call_stream: bad arguments");
    return DG_EINVAL;
  }
  if (h->outstanding) {
    set_error("dg_pipeline_call_stream: submitted steps are outstanding; collect them first");
    return DG_EINVAL;
  }
  int rc;
  const int S = stream_window_len(s);
  StepShape sh = {B};
  if ((rc = dg_seg_dims(h->seg, S, &sh.F, &sh.K))) return rc;
  if (!post_fits(h, post, sh) || s->device != h->seg->device) {
    set_error("dg_pipeline_call_stream: handles were created for other dimensions / devices");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->seg->device));
  if (h->wav.ensure((size_t)B * S * 4) || h->segd.ensure(sh.seg_bytes()) || h->embd.ensure(sh.emb_bytes(h->emb->D)) ||
      h->mapd.ensure(sh.map_bytes()))
    return DG_ECUDA;
  if ((rc = stream_expand(s, B, h->wav.as<float>(), h->st))) return rc;
  const StepOut dev = {h->segd.as<float>(), h->embd.as<float>(), h->mapd.as<int32_t>(), nullptr};
  if ((rc = pipeline_step(h, h->wav.as<float>(), S, sh, dev, h->st, s->rs ? 0 : s->hop))) return rc;
  return call_finish(h, post, sh, plan_host, header_host, turns_host, turn_cap_host, n_turns, seg_host, map_host, nullptr);
}

extern "C" int dg_pipeline_destroy(dg_pipeline* h) {
  delete h;
  return DG_OK;
}

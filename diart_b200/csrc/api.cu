// C ABI of libdiartb200.so (include/diart_b200.h), common part: error state, launch count, profiling, the weight upload
// helpers and the self-tests.  The handles live in api_seg.cu, api_emb.cu, api_cluster.cu, api_stream.cu, api_post.cu and
// api_pipeline.cu.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <sstream>
#include <vector>

#include "host.cuh"

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

int upload_u16(DevBuf& b, const std::vector<uint16_t>& h) {
  if (b.ensure(h.size() * 2)) return -2;
  DG_CUDA(cudaMemcpy(b.p, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  return 0;
}

// float32 [N][K] host weights -> zero-padded planes [Npad][K]
int upload_split(WeightPlanes& w, const std::vector<float>& w_nk, int N, int Npad, int K) {
  std::vector<uint16_t> h((size_t)Npad * K), l((size_t)Npad * K);
  w.scale = weight_plane_scale(w_nk.data(), (size_t)N * K);
  w.Npad = Npad;
  w.K = K;
  split_weights_host(w_nk.data(), N, Npad, K, h.data(), l.data(), w.scale);
  return (upload_u16(w.hi, h) || upload_u16(w.lo, l)) ? DG_ECUDA : 0;
}

// points `t` at its weight planes; the launch's taps and channels (KW, Cin) must span exactly the planes' K
int set_weights(TcGemm& t, const WeightPlanes& w) {
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

int upload(DevBuf& b, const std::vector<float>& h) {
  if (b.ensure(h.size() * sizeof(float))) return -2;
  DG_CUDA(cudaMemcpy(b.p, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

}  // namespace dg

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
  if (M < 1 || Cin < 16 || Cin % 16 || KW < 1 || N % 4 || !max_abs_diff || !out_rms) {
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

// Runs one seeded shifted-window GEMM with epilogue `epi` (0..5) under SM caps of 0 (none), 1, 3 and 7 and sets *equal to 1
// if every output is byte-equal across the four grids: float32 rows, hi/lo planes, pooling partial sums.  Per epilogue:
// 3 = 3 x 3 Conv2d (KW must be 9; `dil` = Hp, M = whole padded maps) with residual planes and ReLU -> hi/lo planes;
// 4 = statistics pooling of 3 speakers over items of 296 rows; 5 = MaxPool1d(3) over items of 888 rows (M a multiple of it).
extern "C" int dg_selftest_gemm_tc_grid(int M, int Cin, int KW, int dil, int N, int epi, int* equal) {
  if (M < 1 || Cin % 64 || KW < 1 || KW > 9 || N < 1 || N % 4 || epi < 0 || epi > 5 || !equal ||
      (epi == 3 && (KW != 9 || dil < 3 || M % (dil * dil) || N % 32)) || (epi == 5 && (N > 64 || M % 888))) {
    set_error("dg_selftest_gemm_tc_grid: bad arguments");
    return DG_EINVAL;
  }
  const int K = KW * Cin;
  const int npad = epi == 5 || N == 64 ? 64 : (epi == 3 && N == 32 ? 32 : (N + 127) / 128 * 128);
  const int ldc = epi == 3 ? (N + 31) / 32 * 32 : N;
  const int item_rows = epi == 4 ? 296 : 888, tile_rows = epi == 5 ? gemm_tc_pool3_tile_rows(item_rows) : 128;
  const long long m_tiles = (M + tile_rows - 1) / tile_rows;
  uint32_t seed = 777u;
  auto rnd = [&]() {
    seed = seed * 1664525u + 1013904223u;
    return ((seed >> 8) & 0xFFFF) / 65536.f - 0.5f;
  };
  std::vector<float> A((size_t)M * Cin), Wnk((size_t)N * K), bias(N), bsc(N), bsh(N), res((size_t)M * ldc), pw((size_t)M * 4);
  for (auto& v : A) v = 2.f * rnd();
  for (auto& v : Wnk) v = 0.25f * rnd();
  for (int n = 0; n < N; n++) {
    bias[n] = rnd();
    bsc[n] = 1.f + rnd();
    bsh[n] = rnd();
  }
  for (auto& v : res) v = rnd();
  for (auto& v : pw) v = rnd() + 0.5f;
  // output buffers, in bytes: float32 rows, hi and lo planes, pooling partial sums
  const size_t f32_bytes = epi == 0 || epi == 2 ? (size_t)M * ldc * 4 : (epi == 5 ? (size_t)(M / 3) * ldc * 4 : 0);
  const size_t plane_bytes = epi == 1 || epi == 3 ? (size_t)M * ldc * 2 : 0;
  const size_t part_bytes = epi == 4 ? (size_t)m_tiles * 2 * TC_POOL_SLOTS * N * 4 : (epi == 5 ? (size_t)m_tiles * 2 * TC_POOL3_SLOTS * N * 4 : 0);
  DevBuf dA, dAh, dAl, dB, dS, dH, dRes, dRh, dRl, dPw, dF, dOh, dOl, dPart;
  WeightPlanes dW;
  if (upload(dA, A) || upload(dB, bias) || upload(dS, bsc) || upload(dH, bsh) || upload(dRes, res) || upload(dPw, pw) ||
      upload_split(dW, Wnk, N, npad, K))
    return DG_ECUDA;
  if (dAh.ensure((size_t)M * Cin * 2) || dAl.ensure((size_t)M * Cin * 2) || dRh.ensure((size_t)M * ldc * 2) ||
      dRl.ensure((size_t)M * ldc * 2) || dF.ensure(f32_bytes + 4) || dOh.ensure(plane_bytes + 4) ||
      dOl.ensure(plane_bytes + 4) || dPart.ensure(part_bytes + 4))
    return DG_ECUDA;
  int rc;
  if ((rc = launch_split_ex(dA.as<float>(), M, Cin, Cin, Cin, 0, 1, nullptr, nullptr, dAh.p, dAl.p, nullptr)) ||
      (rc = launch_split_ex(dRes.as<float>(), M, ldc, ldc, ldc, 0, 1, nullptr, nullptr, dRh.p, dRl.p, nullptr)))
    return rc;
  int taps[9];
  for (int j = 0; j < 9; j++) taps[j] = (j / 3 - 1) * dil + (j % 3 - 1);   // Conv2d: (dw - 1) * Hp + (dh - 1)
  TcGemm t{};
  t.A_hi = dAh.p; t.A_lo = dAl.p; t.lda = Cin; t.Cin = Cin; t.KW = KW; t.dil = dil; t.Mtot = M; t.M = M;
  t.N = N; t.bias = dB.as<float>(); t.bn_scale = dS.as<float>(); t.bn_shift = dH.as<float>(); t.ldc = ldc;
  t.epi = epi; t.tag = "selftest_tc_grid";
  t.out_f32 = f32_bytes ? dF.as<float>() : nullptr;
  t.out_hi = plane_bytes ? dOh.p : nullptr;
  t.out_lo = plane_bytes ? dOl.p : nullptr;
  if (epi == 3) {
    t.tap_off = taps; t.Wp = t.Wop = t.Hp = t.Hop = dil; t.relu = 1;
    t.res_hi = dRh.p; t.res_lo = dRl.p;
  }
  if (epi == 4) {
    t.pool_w = dPw.as<float>(); t.pool_part = dPart.as<float>(); t.pool_item_rows = item_rows; t.pool_K = 3; t.pool_T = item_rows;
  }
  if (epi == 5) {
    t.pool_part = dPart.as<float>(); t.pool_item_rows = item_rows; t.pool3_T = item_rows / 3 - 2;
    t.pool3_tile_rows = tile_rows;
  }
  if ((rc = set_weights(t, dW))) return rc;
  std::vector<unsigned char> first, cur;
  *equal = 1;
  const int caps[4] = {0, 1, 3, 7};
  for (int ci = 0; ci < 4; ci++) {
    // unwritten bytes (rows outside a Conv2d map, pooling slots of absent items) compare equal because they stay zero
    DG_CUDA(cudaMemset(dF.p, 0, f32_bytes + 4));
    DG_CUDA(cudaMemset(dOh.p, 0, plane_bytes + 4));
    DG_CUDA(cudaMemset(dOl.p, 0, plane_bytes + 4));
    DG_CUDA(cudaMemset(dPart.p, 0, part_bytes + 4));
    {
      SmLimit cap(caps[ci]);
      if ((rc = launch_gemm_tc(t, nullptr))) return rc;
    }
    DG_CUDA(cudaDeviceSynchronize());
    cur.resize(f32_bytes + 2 * plane_bytes + part_bytes);
    DG_CUDA(cudaMemcpy(cur.data(), dF.p, f32_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(cur.data() + f32_bytes, dOh.p, plane_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(cur.data() + f32_bytes + plane_bytes, dOl.p, plane_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(cur.data() + f32_bytes + 2 * plane_bytes, dPart.p, part_bytes, cudaMemcpyDeviceToHost));
    if (ci == 0)
      first.swap(cur);
    else if (cur != first)
      *equal = 0;
  }
  return DG_OK;
}

// Sets bit r of *ok_shifts when a wgmma whose A descriptor starts r = 0..8 rows into a 64B-swizzled TMA tile computes the
// exact product of rows r..r+63; base_offset_mode 1 also sets the descriptor's matrix base offset to (address >> 7) & 7.
extern "C" int dg_selftest_wgmma_row_shift(int base_offset_mode, unsigned* ok_shifts) {
  if (base_offset_mode < 0 || base_offset_mode > 1 || !ok_shifts) {
    set_error("dg_selftest_wgmma_row_shift: bad arguments");
    return DG_EINVAL;
  }
  return selftest_wgmma_row_shift(base_offset_mode, ok_shifts) ? DG_ECUDA : DG_OK;
}

// Sets bit r of *ok_shifts when a wgmma whose B descriptor starts r = 0..8 rows into a 64B-swizzled TMA tile computes the
// exact product with rows r..r+63 (the weight-stationary MaxPool3 kernel's time rows); base_offset_mode as above.
extern "C" int dg_selftest_wgmma_b_row_shift(int base_offset_mode, unsigned* ok_shifts) {
  if (base_offset_mode < 0 || base_offset_mode > 1 || !ok_shifts) {
    set_error("dg_selftest_wgmma_b_row_shift: bad arguments");
    return DG_EINVAL;
  }
  return selftest_wgmma_b_row_shift(base_offset_mode, ok_shifts) ? DG_ECUDA : DG_OK;
}

// Runs one seeded Conv1d with the MaxPool1d(3) epilogue (epilogue 5, items of 888 rows, M a multiple of them) through
// launch_gemm_tc, and the same convolution through the float32 reference GEMM (gemm.cu) pooled on the host; reports the
// largest absolute difference of the pooled rows and their scale.  *ws = 1 if the launch took the weight-stationary kernel.
extern "C" int dg_selftest_gemm_tc_pool3_simt(int M, int Cin, int KW, int dil, int N, float* max_abs_diff, float* out_rms,
                                              int* ws) {
  if (M < 888 || M % 888 || Cin < 16 || Cin % 16 || Cin > 128 || KW < 2 || KW > 9 || dil < 1 || N < 1 || N > 64 || N % 4 ||
      !max_abs_diff || !out_rms || !ws) {
    set_error("dg_selftest_gemm_tc_pool3_simt: bad arguments");
    return DG_EINVAL;
  }
  const int K = KW * Cin, item_rows = 888, tile_rows = gemm_tc_pool3_tile_rows(item_rows);
  const long long m_tiles = (M + tile_rows - 1) / tile_rows, tail = (long long)(KW - 1) * dil;
  uint32_t seed = 4242u;
  auto rnd = [&]() {
    seed = seed * 1664525u + 1013904223u;
    return ((seed >> 8) & 0xFFFF) / 65536.f - 0.5f;
  };
  // the reference reads KW - 1 taps past M: zero rows, as TMA fills them
  std::vector<float> A((size_t)(M + tail) * Cin, 0.f), Wkn((size_t)K * N), Wnk((size_t)N * K), bias(N);
  for (size_t i = 0; i < (size_t)M * Cin; i++) A[i] = 2.f * rnd();
  for (int k = 0; k < K; k++)
    for (int n = 0; n < N; n++) Wkn[(size_t)k * N + n] = Wnk[(size_t)n * K + k] = 0.25f * rnd();
  for (auto& v : bias) v = rnd();
  DevBuf dA, dWkn, dB, dAh, dAl, dC0, dP, dPart;
  WeightPlanes dW;
  if (upload(dA, A) || upload(dWkn, Wkn) || upload(dB, bias) || upload_split(dW, Wnk, N, 64, K)) return DG_ECUDA;
  if (dAh.ensure((size_t)M * Cin * 2) || dAl.ensure((size_t)M * Cin * 2) || dC0.ensure((size_t)M * N * 4) ||
      dP.ensure((size_t)(M / 3) * N * 4) || dPart.ensure((size_t)m_tiles * 2 * TC_POOL3_SLOTS * N * 4))
    return DG_ECUDA;
  int rc;
  GemmArgs g{};
  g.A = dA.as<float>(); g.lda = Cin; g.Cin = Cin; g.KW = KW; g.dil = dil; g.Mtot = M + tail; g.M = M;
  g.W = dWkn.as<float>(); g.ldw = N; g.N = N; g.bias = dB.as<float>(); g.C = dC0.as<float>(); g.ldc = N; g.epi = EPI_BIAS;
  g.tag = "selftest_simt";
  if ((rc = launch_gemm(g, nullptr))) return rc;
  if ((rc = launch_split_ex(dA.as<float>(), M, Cin, Cin, Cin, 0, 1, nullptr, nullptr, dAh.p, dAl.p, nullptr))) return rc;
  TcGemm t{};
  t.A_hi = dAh.p; t.A_lo = dAl.p; t.lda = Cin; t.Cin = Cin; t.KW = KW; t.dil = dil; t.Mtot = M; t.M = M;
  t.N = N; t.bias = dB.as<float>(); t.out_f32 = dP.as<float>(); t.ldc = N; t.epi = 5; t.tag = "selftest_tc_pool3";
  t.pool_part = dPart.as<float>(); t.pool_item_rows = item_rows; t.pool3_T = item_rows / 3 - 2; t.pool3_tile_rows = tile_rows;
  if ((rc = set_weights(t, dW))) return rc;
  *ws = gemm_tc_ws(t) ? 1 : 0;
  if ((rc = launch_gemm_tc(t, nullptr))) return rc;
  DG_CUDA(cudaDeviceSynchronize());
  std::vector<float> c0((size_t)M * N), p1((size_t)(M / 3) * N);
  DG_CUDA(cudaMemcpy(c0.data(), dC0.p, c0.size() * 4, cudaMemcpyDeviceToHost));
  DG_CUDA(cudaMemcpy(p1.data(), dP.p, p1.size() * 4, cudaMemcpyDeviceToHost));
  double md = 0, ss = 0;
  for (long long r = 0; r < M / 3; r++)
    for (int n = 0; n < N; n++) {
      const float* x = &c0[(size_t)(3 * r) * N + n];
      const double ref = std::max(std::max(x[0], x[N]), x[2 * N]);
      const double d = fabs(ref - (double)p1[(size_t)r * N + n]);
      if (!(d <= md)) md = d;     // NaN-propagating max
      ss += ref * ref;
    }
  *max_abs_diff = (float)md;
  *out_rms = (float)sqrt(ss / p1.size());
  return DG_OK;
}

// Runs one seeded Conv1d GEMM (epilogue 0, 1, 2 or 5) through the halo operand mode, under no SM cap and under a cap of 3
// SMs, and through the tap-box mode, and sets *equal = 1 if all three wrote the same bytes: float32 rows, hi/lo planes,
// pooling partial sums.  A Cin that is not a multiple of 64 (SincNet's 80) has no tap-box form: the reference then reads
// the taps folded into K = KW * Cin rounded up to 64 through an overlapping-row view (dil must be 1), with zero weights
// past KW * Cin.  *halo = 1 if the launch took the halo mode.  Epilogue 5 pools items of 888 rows (M a multiple of it).
extern "C" int dg_selftest_gemm_tc_halo(int M, int Cin, int KW, int dil, int N, int epi, int* equal, int* halo) {
  const bool folded = Cin % 64 != 0;
  if (M < 1 || Cin < 16 || Cin % 16 || Cin > 128 || KW < 2 || KW > 9 || dil < 1 || N < 1 || N % 4 ||
      (epi != 0 && epi != 1 && epi != 2 && epi != 5) || (epi == 1 && N % 32) || (epi == 5 && (N > 64 || M % 888)) ||
      (folded && dil != 1) || !equal || !halo) {
    set_error("dg_selftest_gemm_tc_halo: bad arguments");
    return DG_EINVAL;
  }
  const int K = KW * Cin, Kf = folded ? (K + 63) / 64 * 64 : K;
  const int npad = epi == 5 || N == 64 ? 64 : (N + 127) / 128 * 128;
  const int item_rows = 888, tile_rows = epi == 5 ? gemm_tc_pool3_tile_rows(item_rows) : 128;
  const long long m_tiles = (M + tile_rows - 1) / tile_rows;
  const long long tail = 64;   // zero rows after M: the folded view reads up to Kf / Cin rows past its own
  uint32_t seed = 9090u;
  auto rnd = [&]() {
    seed = seed * 1664525u + 1013904223u;
    return ((seed >> 8) & 0xFFFF) / 65536.f - 0.5f;
  };
  std::vector<float> A((size_t)(M + tail) * Cin, 0.f), Wnk((size_t)N * K), Wf((size_t)N * Kf, 0.f), bias(N), bsc(N), bsh(N);
  for (size_t i = 0; i < (size_t)M * Cin; i++) A[i] = 2.f * rnd();
  for (auto& v : Wnk) v = 0.25f * rnd();
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) Wf[(size_t)n * Kf + k] = Wnk[(size_t)n * K + k];
  for (int n = 0; n < N; n++) {
    bias[n] = rnd();
    bsc[n] = 1.f + rnd();
    bsh[n] = rnd();
  }
  const size_t f32_bytes = epi == 0 || epi == 2 ? (size_t)M * N * 4 : (epi == 5 ? (size_t)(M / 3) * N * 4 : 0);
  const size_t plane_bytes = epi == 1 ? (size_t)M * N * 2 : 0;
  const size_t part_bytes = epi == 5 ? (size_t)m_tiles * 2 * TC_POOL3_SLOTS * N * 4 : 0;
  DevBuf dA, dAh, dAl, dB, dS, dH, dF, dOh, dOl, dPart;
  WeightPlanes dW, dWf;
  if (upload(dA, A) || upload(dB, bias) || upload(dS, bsc) || upload(dH, bsh) || upload_split(dW, Wnk, N, npad, K) ||
      upload_split(dWf, Wf, N, npad, Kf))
    return DG_ECUDA;
  if (dAh.ensure((size_t)(M + tail) * Cin * 2) || dAl.ensure((size_t)(M + tail) * Cin * 2) || dF.ensure(f32_bytes + 4) ||
      dOh.ensure(plane_bytes + 4) || dOl.ensure(plane_bytes + 4) || dPart.ensure(part_bytes + 4))
    return DG_ECUDA;
  int rc;
  if ((rc = launch_split_ex(dA.as<float>(), M + tail, Cin, Cin, Cin, 0, 1, nullptr, nullptr, dAh.p, dAl.p, nullptr))) return rc;
  TcGemm t{};
  t.A_hi = dAh.p; t.A_lo = dAl.p; t.lda = Cin; t.Cin = Cin; t.KW = KW; t.dil = dil; t.Mtot = M; t.M = M;
  t.N = N; t.bias = dB.as<float>(); t.bn_scale = dS.as<float>(); t.bn_shift = dH.as<float>(); t.ldc = N;
  t.epi = epi; t.tag = "selftest_tc_halo";
  t.out_f32 = f32_bytes ? dF.as<float>() : nullptr;
  t.out_hi = plane_bytes ? dOh.p : nullptr;
  t.out_lo = plane_bytes ? dOl.p : nullptr;
  if (epi == 5) {
    t.pool_part = dPart.as<float>(); t.pool_item_rows = item_rows; t.pool3_T = item_rows / 3 - 2;
    t.pool3_tile_rows = tile_rows;
  }
  if ((rc = set_weights(t, dW))) return rc;
  *halo = gemm_tc_halo(t) ? 1 : 0;
  TcGemm ref = t;
  ref.tap_boxes = 1;
  if (folded) {
    ref.Cin = Kf;
    ref.KW = 1;
    if ((rc = set_weights(ref, dWf))) return rc;
  }
  std::vector<unsigned char> first, cur;
  *equal = 1;
  for (int run = 0; run < 3; run++) {   // halo, halo on 3 SMs, tap boxes
    DG_CUDA(cudaMemset(dF.p, 0, f32_bytes + 4));
    DG_CUDA(cudaMemset(dOh.p, 0, plane_bytes + 4));
    DG_CUDA(cudaMemset(dOl.p, 0, plane_bytes + 4));
    DG_CUDA(cudaMemset(dPart.p, 0, part_bytes + 4));
    {
      SmLimit cap(run == 1 ? 3 : 0);
      if ((rc = launch_gemm_tc(run == 2 ? ref : t, nullptr))) return rc;
    }
    DG_CUDA(cudaDeviceSynchronize());
    cur.resize(f32_bytes + 2 * plane_bytes + part_bytes);
    DG_CUDA(cudaMemcpy(cur.data(), dF.p, f32_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(cur.data() + f32_bytes, dOh.p, plane_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(cur.data() + f32_bytes + plane_bytes, dOl.p, plane_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(cur.data() + f32_bytes + 2 * plane_bytes, dPart.p, part_bytes, cudaMemcpyDeviceToHost));
    if (run == 0)
      first.swap(cur);
    else if (cur != first)
      *equal = 0;
  }
  return DG_OK;
}

// Runs one seeded GEMM (one tap, epilogue 0, 1 or 2) twice: into outputs of pitch N, and into outputs of pitch N + 40 with
// 130 guard rows after M, all bytes preset to a sentinel.  Sets *outside_unchanged = 1 if the second run changed no byte
// outside rows [0, M) x columns [0, N), *equal = 1 if inside them it wrote the first run's bytes, and *refused = 1 if the
// launcher rejects, with DG_EINVAL and without writing, an output base 4 (float32) or 2 (planes) bytes off 16-byte
// alignment and a pitch whose byte size is not a multiple of 16.
extern "C" int dg_selftest_gemm_tc_bounds(int M, int Cin, int N, int epi, int* outside_unchanged, int* equal, int* refused) {
  const bool planes = epi == 1;
  if (M < 1 || Cin < 64 || Cin % 64 || N < 1 || N % (planes ? 32 : 4) || epi < 0 || epi > 2 || !outside_unchanged || !equal ||
      !refused) {
    set_error("dg_selftest_gemm_tc_bounds: bad arguments");
    return DG_EINVAL;
  }
  const int npad = N <= 64 && epi == 0 ? 64 : (N + 127) / 128 * 128, esize = planes ? 2 : 4;   // 64-wide tiles: epi 0 only
  const int ldc = N + 40;
  const long long rows = (long long)M + 130;
  uint32_t seed = 4242u;
  auto rnd = [&]() {
    seed = seed * 1664525u + 1013904223u;
    return ((seed >> 8) & 0xFFFF) / 65536.f - 0.5f;
  };
  std::vector<float> A((size_t)M * Cin), Wnk((size_t)N * Cin), bias(N), bsc(N), bsh(N);
  for (auto& v : A) v = 2.f * rnd();
  for (auto& v : Wnk) v = 0.25f * rnd();
  for (int n = 0; n < N; n++) {
    bias[n] = rnd();
    bsc[n] = 1.f + rnd();
    bsh[n] = rnd();
  }
  const size_t dense_bytes = (size_t)M * N * esize, wide_bytes = (size_t)rows * ldc * esize + 16;
  DevBuf dA, dAh, dAl, dB, dS, dH, dD0, dD1, dW0, dW1;
  WeightPlanes dW;
  if (upload(dA, A) || upload(dB, bias) || upload(dS, bsc) || upload(dH, bsh) || upload_split(dW, Wnk, N, npad, Cin) ||
      dAh.ensure((size_t)M * Cin * 2) || dAl.ensure((size_t)M * Cin * 2) || dD0.ensure(dense_bytes) ||
      dD1.ensure(dense_bytes) || dW0.ensure(wide_bytes) || dW1.ensure(wide_bytes))
    return DG_ECUDA;
  int rc;
  if ((rc = launch_split_ex(dA.as<float>(), M, Cin, Cin, Cin, 0, 1, nullptr, nullptr, dAh.p, dAl.p, nullptr))) return rc;
  TcGemm t{};
  t.A_hi = dAh.p; t.A_lo = dAl.p; t.lda = Cin; t.Cin = Cin; t.KW = 1; t.dil = 1; t.Mtot = M; t.M = M;
  t.N = N; t.bias = dB.as<float>(); t.bn_scale = dS.as<float>(); t.bn_shift = dH.as<float>();
  t.epi = epi; t.tag = "selftest_tc_bounds";
  if ((rc = set_weights(t, dW))) return rc;
  // output 0 (float32 rows or hi plane) and 1 (lo plane) at `off` bytes into the buffers, pitch `ld`
  auto point = [&](DevBuf& o0, DevBuf& o1, size_t off, int ld) {
    unsigned char* b0 = static_cast<unsigned char*>(o0.p) + off;
    unsigned char* b1 = static_cast<unsigned char*>(o1.p) + off;
    t.out_f32 = planes ? nullptr : reinterpret_cast<float*>(b0);
    t.out_hi = planes ? b0 : nullptr;
    t.out_lo = planes ? b1 : nullptr;
    t.ldc = ld;
  };
  const unsigned char SENTINEL = 0xA5;
  DG_CUDA(cudaMemset(dW0.p, SENTINEL, wide_bytes));
  DG_CUDA(cudaMemset(dW1.p, SENTINEL, wide_bytes));
  point(dD0, dD1, 0, N);
  if ((rc = launch_gemm_tc(t, nullptr))) return rc;
  point(dW0, dW1, 0, ldc);
  if ((rc = launch_gemm_tc(t, nullptr))) return rc;
  // refusals: base off alignment, pitch off 16 bytes (both leave the sentinel in place)
  point(dW0, dW1, (size_t)esize, ldc);
  const int rc_base = launch_gemm_tc(t, nullptr);
  point(dW0, dW1, 0, ldc + (planes ? 4 : 2));
  const int rc_pitch = launch_gemm_tc(t, nullptr);
  DG_CUDA(cudaDeviceSynchronize());
  const int n_out = planes ? 2 : 1;
  std::vector<unsigned char> dense(dense_bytes), wide(wide_bytes);
  *outside_unchanged = 1;
  *equal = 1;
  for (int o = 0; o < n_out; o++) {
    DG_CUDA(cudaMemcpy(dense.data(), (o ? dD1 : dD0).p, dense_bytes, cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(wide.data(), (o ? dW1 : dW0).p, wide_bytes, cudaMemcpyDeviceToHost));
    const size_t row_bytes = (size_t)N * esize, pitch = (size_t)ldc * esize;
    for (long long r = 0; r < rows; r++) {
      const unsigned char* w = wide.data() + r * pitch;
      const bool inside = r < M;
      if (inside && memcmp(w, dense.data() + r * row_bytes, row_bytes)) *equal = 0;
      for (size_t b = inside ? row_bytes : 0; b < pitch; b++)
        if (w[b] != SENTINEL) *outside_unchanged = 0;
    }
    for (size_t b = (size_t)rows * pitch; b < wide_bytes; b++)
      if (wide[b] != SENTINEL) *outside_unchanged = 0;
  }
  *refused = rc_base == DG_EINVAL && rc_pitch == DG_EINVAL;
  return DG_OK;
}

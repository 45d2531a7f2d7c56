// C ABI of libdiartb200.so (include/diart_b200.h), common part: error state, launch count, profiling, the weight upload
// helpers and the self-tests.  The handles live in api_seg.cu, api_emb.cu, api_cluster.cu, api_stream.cu, api_post.cu and
// api_pipeline.cu.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <initializer_list>
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

// ---- shared by the gemm_tc self-tests
// Seeded operands of a shifted-window GEMM, drawn in one order: A [M][Cin] (amplitude 2, then `tail_rows` zero rows), W in
// [K][N] order, then bias, BatchNorm scale and shift per column.  A caller draws its extras from rnd() afterwards.  On the
// device: A in float32 and as fp16 hi/lo planes (all M + tail_rows rows), W as weight planes of Npad rows, the three vectors.
struct GemmFixture {
  int M = 0, Cin = 0, KW = 0, N = 0;
  long long rows = 0;
  uint32_t seed = 0;
  std::vector<float> W;   // [K][N]
  DevBuf dA, dAh, dAl, dB, dS, dH;
  WeightPlanes planes;

  float rnd() {
    seed = seed * 1664525u + 1013904223u;
    return ((seed >> 8) & 0xFFFF) / 65536.f - 0.5f;
  }
  int init(int M_, int Cin_, int KW_, int N_, int npad, uint32_t seed_, long long tail_rows = 0) {
    M = M_, Cin = Cin_, KW = KW_, N = N_, rows = M + tail_rows, seed = seed_;
    const int K = KW * Cin;
    std::vector<float> A((size_t)rows * Cin, 0.f), Wnk((size_t)N * K), bias(N), bsc(N), bsh(N);
    W.resize((size_t)K * N);
    for (size_t i = 0; i < (size_t)M * Cin; i++) A[i] = 2.f * rnd();
    for (auto& v : W) v = 0.25f * rnd();
    for (int n = 0; n < N; n++) {
      bias[n] = rnd();
      bsc[n] = 1.f + rnd();
      bsh[n] = rnd();
    }
    for (int k = 0; k < K; k++)
      for (int n = 0; n < N; n++) Wnk[(size_t)n * K + k] = W[(size_t)k * N + n];
    if (upload(dA, A) || upload(dB, bias) || upload(dS, bsc) || upload(dH, bsh) || upload_split(planes, Wnk, N, npad, K) ||
        dAh.ensure((size_t)rows * Cin * 2) || dAl.ensure((size_t)rows * Cin * 2))
      return DG_ECUDA;
    return launch_split_ex(dA.as<float>(), rows, Cin, Cin, Cin, 0, 1, nullptr, nullptr, dAh.p, dAl.p, nullptr);
  }
  // `t` over these operands with epilogue `epi`, output pitch N and no outputs yet
  int gemm(TcGemm& t, int dil, int epi, const char* tag) const {
    t = TcGemm{};
    t.A_hi = dAh.p; t.A_lo = dAl.p; t.lda = Cin; t.Cin = Cin; t.KW = KW; t.dil = dil; t.Mtot = M; t.M = M;
    t.N = N; t.bias = dB.as<float>(); t.bn_scale = dS.as<float>(); t.bn_shift = dH.as<float>(); t.ldc = N;
    t.epi = epi; t.tag = tag;
    return set_weights(t, planes);
  }
  // the float32 reference GEMM (gemm.cu) over all rows of A: bias (epi 0) or bias + LeakyReLU + BatchNorm -> c [M][N]
  int simt(int dil, int epi, std::vector<float>& c) const {
    DevBuf dW, dC;
    if (upload(dW, W) || dC.ensure((size_t)M * N * 4)) return DG_ECUDA;
    GemmArgs g{};
    g.A = dA.as<float>(); g.lda = Cin; g.Cin = Cin; g.KW = KW; g.dil = dil; g.Mtot = rows; g.M = M;
    g.W = dW.as<float>(); g.ldw = N; g.N = N; g.bias = dB.as<float>(); g.bn_scale = dS.as<float>();
    g.bn_shift = dH.as<float>(); g.C = dC.as<float>(); g.ldc = N; g.epi = epi == 0 ? EPI_BIAS : EPI_BIAS_LEAKY_BN;
    g.tag = "selftest_simt";
    int rc;
    if ((rc = launch_gemm(g, nullptr))) return rc;
    c.resize((size_t)M * N);
    DG_CUDA(cudaMemcpy(c.data(), dC.p, c.size() * 4, cudaMemcpyDeviceToHost));
    return 0;
  }
};

// The outputs of a TcGemm: float32 rows, hi plane, lo plane and pooling partial sums, each sized by the epilogue (empty if
// it writes none).
struct GemmOutputs {
  DevBuf buf[4];
  size_t bytes[4] = {};
  // sizes the outputs from t's epilogue, rows, pitch and columns and the rows an m-tile advances by, and points t at them
  int attach(TcGemm& t, int tile_rows) {
    const int epi = t.epi;
    const size_t m_tiles = (t.M + tile_rows - 1) / tile_rows, cells = (size_t)(epi == 5 ? t.M / 3 : t.M) * t.ldc;
    bytes[0] = epi == 1 || epi == 3 || epi == 4 ? 0 : cells * 4;   // the launcher runs an unknown epilogue as 2
    bytes[1] = bytes[2] = epi == 1 || epi == 3 ? cells * 2 : 0;
    bytes[3] = epi == 4 || epi == 5 ? m_tiles * 2 * (epi == 4 ? TC_POOL_SLOTS : TC_POOL3_SLOTS) * t.N * 4 : 0;
    for (int i = 0; i < 4; i++)
      if (buf[i].ensure(bytes[i] + 4)) return DG_ECUDA;
    t.out_f32 = bytes[0] ? buf[0].as<float>() : nullptr;
    t.out_hi = bytes[1] ? buf[1].p : nullptr;
    t.out_lo = bytes[2] ? buf[2].p : nullptr;
    t.pool_part = bytes[3] ? buf[3].as<float>() : nullptr;
    return 0;
  }
  // clears the outputs, runs `t` on at most `sm_cap` SMs (0: all) and returns what it wrote, the four outputs back to back;
  // bytes it leaves unwritten (rows outside a Conv2d map, pooling slots of absent items) read as zero
  int run(const TcGemm& t, int sm_cap, std::vector<unsigned char>& out) {
    for (int i = 0; i < 4; i++) DG_CUDA(cudaMemset(buf[i].p, 0, bytes[i] + 4));
    int rc;
    {
      SmLimit cap(sm_cap);
      if ((rc = launch_gemm_tc(t, nullptr))) return rc;
    }
    DG_CUDA(cudaDeviceSynchronize());
    out.resize(bytes[0] + bytes[1] + bytes[2] + bytes[3]);
    size_t at = 0;
    for (int i = 0; i < 4; at += bytes[i++]) DG_CUDA(cudaMemcpy(out.data() + at, buf[i].p, bytes[i], cudaMemcpyDeviceToHost));
    return 0;
  }
  // runs each (launch, SM cap) in turn and sets *equal = 1 if all of them wrote the same bytes
  int equal_runs(std::initializer_list<std::pair<const TcGemm*, int>> runs, int* equal) {
    std::vector<unsigned char> first, cur;
    *equal = 1;
    int rc;
    for (const auto& r : runs) {
      if ((rc = run(*r.first, r.second, cur))) return rc;
      if (first.empty())
        first.swap(cur);
      else if (cur != first)
        *equal = 0;
    }
    return 0;
  }
};

// Runs the same shifted-window GEMM through the float32 reference kernel (gemm.cu) and through the wgmma split-precision
// kernel on seeded random data and reports the largest absolute difference and the output scale.
extern "C" int dg_selftest_gemm_tc(int M, int Cin, int KW, int dil, int N, int epi, float* max_abs_diff,
                                   float* out_rms) {
  if (M < 1 || Cin < 16 || Cin % 16 || KW < 1 || N % 4 || !max_abs_diff || !out_rms) {
    set_error("dg_selftest_gemm_tc: bad arguments");
    return DG_EINVAL;
  }
  GemmFixture f;
  TcGemm t;
  GemmOutputs o;
  std::vector<float> c0;
  std::vector<unsigned char> out;
  int rc;
  if ((rc = f.init(M, Cin, KW, N, N == 64 ? 64 : (N + 255) / 256 * 256, 12345u)) || (rc = f.simt(dil, epi, c0)) ||
      (rc = f.gemm(t, dil, epi, "selftest_tc")) || (rc = o.attach(t, 128)) || (rc = o.run(t, 0, out)))
    return rc;
  const size_t cells = (size_t)M * N;
  std::vector<float> c1(cells);
  std::vector<uint16_t> hl(epi == 1 ? 2 * cells : 0);   // epi 1: hi plane, then lo plane
  memcpy(epi == 1 ? (void*)hl.data() : (void*)c1.data(), out.data(), std::min(out.size(), cells * 4));
  if (epi == 1)
    for (size_t i = 0; i < cells; i++) c1[i] = host_h16_to_f32(hl[i]) + host_h16_to_f32(hl[cells + i]);
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
        fprintf(stderr, "   row %zu col %zu: simt %g, planes hi 0x%04x lo 0x%04x\n", i / N, i % N, c0[i], hl[i], hl[cells + i]);
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
  const int npad = epi == 5 || N == 64 ? 64 : (epi == 3 && N == 32 ? 32 : (N + 127) / 128 * 128);
  const int ldc = epi == 3 ? (N + 31) / 32 * 32 : N;
  const int item_rows = epi == 4 ? 296 : 888, tile_rows = epi == 5 ? gemm_tc_pool3_tile_rows(item_rows) : 128;
  GemmFixture f;
  int rc;
  if ((rc = f.init(M, Cin, KW, N, npad, 777u))) return rc;
  std::vector<float> res((size_t)M * ldc), pw((size_t)M * 4);
  for (auto& v : res) v = f.rnd();
  for (auto& v : pw) v = f.rnd() + 0.5f;
  DevBuf dRes, dRh, dRl, dPw;
  if (upload(dRes, res) || upload(dPw, pw) || dRh.ensure((size_t)M * ldc * 2) || dRl.ensure((size_t)M * ldc * 2))
    return DG_ECUDA;
  if ((rc = launch_split_ex(dRes.as<float>(), M, ldc, ldc, ldc, 0, 1, nullptr, nullptr, dRh.p, dRl.p, nullptr))) return rc;
  int taps[9];
  for (int j = 0; j < 9; j++) taps[j] = (j / 3 - 1) * dil + (j % 3 - 1);   // Conv2d: (dw - 1) * Hp + (dh - 1)
  TcGemm t;
  if ((rc = f.gemm(t, dil, epi, "selftest_tc_grid"))) return rc;
  t.ldc = ldc;
  if (epi == 3) {
    t.tap_off = taps; t.Wp = t.Wop = t.Hp = t.Hop = dil; t.relu = 1;
    t.res_hi = dRh.p; t.res_lo = dRl.p;
  }
  if (epi == 4) {
    t.pool_w = dPw.as<float>(); t.pool_item_rows = item_rows; t.pool_K = 3; t.pool_T = item_rows;
  }
  if (epi == 5) {
    t.pool_item_rows = item_rows; t.pool3_T = item_rows / 3 - 2; t.pool3_tile_rows = tile_rows;
  }
  GemmOutputs o;
  if (o.attach(t, tile_rows)) return DG_ECUDA;
  return o.equal_runs({{&t, 0}, {&t, 1}, {&t, 3}, {&t, 7}}, equal);
}

// Sets bit r of *ok_shifts when a wgmma whose A descriptor (dg_selftest_wgmma_row_shift) or B descriptor
// (dg_selftest_wgmma_b_row_shift: the weight-stationary MaxPool3 kernel's time rows) starts r = 0..8 rows into a 64B-swizzled
// TMA tile computes the exact product with rows r..r+63; base_offset_mode 1 also sets the descriptor's matrix base offset
// to (address >> 7) & 7.
static int row_shift(const char* who, bool shift_b, int base_offset_mode, unsigned* ok_shifts) {
  if (base_offset_mode < 0 || base_offset_mode > 1 || !ok_shifts) {
    set_error(std::string(who) + ": bad arguments");
    return DG_EINVAL;
  }
  return selftest_wgmma_row_shift(shift_b, base_offset_mode, ok_shifts) ? DG_ECUDA : DG_OK;
}
extern "C" int dg_selftest_wgmma_row_shift(int base_offset_mode, unsigned* ok_shifts) {
  return row_shift("dg_selftest_wgmma_row_shift", false, base_offset_mode, ok_shifts);
}
extern "C" int dg_selftest_wgmma_b_row_shift(int base_offset_mode, unsigned* ok_shifts) {
  return row_shift("dg_selftest_wgmma_b_row_shift", true, base_offset_mode, ok_shifts);
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
  const int item_rows = 888, tile_rows = gemm_tc_pool3_tile_rows(item_rows);
  GemmFixture f;
  TcGemm t;
  GemmOutputs o;
  std::vector<float> c0;
  std::vector<unsigned char> out;
  int rc;
  // the reference reads KW - 1 taps past M: zero rows, as TMA fills them
  if ((rc = f.init(M, Cin, KW, N, 64, 4242u, (long long)(KW - 1) * dil)) || (rc = f.simt(dil, 0, c0)) ||
      (rc = f.gemm(t, dil, 5, "selftest_tc_pool3")))
    return rc;
  t.pool_item_rows = item_rows; t.pool3_T = item_rows / 3 - 2; t.pool3_tile_rows = tile_rows;
  if (o.attach(t, tile_rows)) return DG_ECUDA;
  *ws = gemm_tc_ws(t) ? 1 : 0;
  if ((rc = o.run(t, 0, out))) return rc;
  std::vector<float> p1((size_t)(M / 3) * N);
  memcpy(p1.data(), out.data(), p1.size() * 4);
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
  GemmFixture f;
  TcGemm t;
  GemmOutputs o;
  int rc;
  // 64 zero rows after M: the folded view reads up to Kf / Cin rows past its own
  if ((rc = f.init(M, Cin, KW, N, npad, 9090u, 64)) || (rc = f.gemm(t, dil, epi, "selftest_tc_halo"))) return rc;
  if (epi == 5) {
    t.pool_item_rows = item_rows; t.pool3_T = item_rows / 3 - 2; t.pool3_tile_rows = tile_rows;
  }
  if (o.attach(t, tile_rows)) return DG_ECUDA;
  *halo = gemm_tc_halo(t) ? 1 : 0;
  TcGemm ref = t;
  ref.tap_boxes = 1;
  WeightPlanes wf;
  if (folded) {
    std::vector<float> Wf((size_t)N * Kf, 0.f);
    for (int k = 0; k < K; k++)
      for (int n = 0; n < N; n++) Wf[(size_t)n * Kf + k] = f.W[(size_t)k * N + n];
    if (upload_split(wf, Wf, N, npad, Kf)) return DG_ECUDA;
    ref.Cin = Kf;
    ref.KW = 1;
    if ((rc = set_weights(ref, wf))) return rc;
  }
  return o.equal_runs({{&t, 0}, {&t, 3}, {&ref, 0}}, equal);   // halo, halo on 3 SMs, tap boxes
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
  const size_t dense_bytes = (size_t)M * N * esize, wide_bytes = (size_t)rows * ldc * esize + 16;
  GemmFixture f;
  TcGemm t;
  GemmOutputs o;
  std::vector<unsigned char> dense;   // pitch N: float32 rows, or the hi plane and then the lo plane
  int rc;
  if ((rc = f.init(M, Cin, 1, N, npad, 4242u)) || (rc = f.gemm(t, 1, epi, "selftest_tc_bounds")) || (rc = o.attach(t, 128)) ||
      (rc = o.run(t, 0, dense)))
    return rc;
  DevBuf dW0, dW1;
  if (dW0.ensure(wide_bytes) || dW1.ensure(wide_bytes)) return DG_ECUDA;
  // output 0 (float32 rows or hi plane) and 1 (lo plane) at `off` bytes into the wide buffers, pitch `ld`
  auto point = [&](size_t off, int ld) {
    unsigned char* b0 = static_cast<unsigned char*>(dW0.p) + off;
    unsigned char* b1 = static_cast<unsigned char*>(dW1.p) + off;
    t.out_f32 = planes ? nullptr : reinterpret_cast<float*>(b0);
    t.out_hi = planes ? b0 : nullptr;
    t.out_lo = planes ? b1 : nullptr;
    t.ldc = ld;
  };
  const unsigned char SENTINEL = 0xA5;
  DG_CUDA(cudaMemset(dW0.p, SENTINEL, wide_bytes));
  DG_CUDA(cudaMemset(dW1.p, SENTINEL, wide_bytes));
  point(0, ldc);
  if ((rc = launch_gemm_tc(t, nullptr))) return rc;
  // refusals: base off alignment, pitch off 16 bytes (both leave the sentinel in place)
  point((size_t)esize, ldc);
  const int rc_base = launch_gemm_tc(t, nullptr);
  point(0, ldc + (planes ? 4 : 2));
  const int rc_pitch = launch_gemm_tc(t, nullptr);
  DG_CUDA(cudaDeviceSynchronize());
  const int n_out = planes ? 2 : 1;
  std::vector<unsigned char> wide(wide_bytes);
  *outside_unchanged = 1;
  *equal = 1;
  for (int i = 0; i < n_out; i++) {
    DG_CUDA(cudaMemcpy(wide.data(), (i ? dW1 : dW0).p, wide_bytes, cudaMemcpyDeviceToHost));
    const size_t row_bytes = (size_t)N * esize, pitch = (size_t)ldc * esize;
    for (long long r = 0; r < rows; r++) {
      const unsigned char* w = wide.data() + r * pitch;
      const bool inside = r < M;
      if (inside && memcmp(w, dense.data() + i * dense_bytes + r * row_bytes, row_bytes)) *equal = 0;
      for (size_t b = inside ? row_bytes : 0; b < pitch; b++)
        if (w[b] != SENTINEL) *outside_unchanged = 0;
    }
    for (size_t b = (size_t)rows * pitch; b < wide_bytes; b++)
      if (wide[b] != SENTINEL) *outside_unchanged = 0;
  }
  *refused = rc_base == DG_EINVAL && rc_pitch == DG_EINVAL;
  return DG_OK;
}

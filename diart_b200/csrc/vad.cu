// Voice activity detection sweep on the device: the reference tunes VoiceActivityDetection's only hyper-parameter, tau_active,
// by running the whole pipeline once per trial (Optimizer.objective -> Benchmark, reference src/diart/optim.py:98-122).  The
// threshold is read by Binarize alone (blocks/vad.py:150-180), so here the speech curve -- the max over the local speakers
// (vad.py:145-148) aggregated over the `latency / step` most recent chunks -- is computed once per dataset and every trial
// only compares it with its own threshold.
//
//   vad_curve      one CTA per chunk: max over the K local speakers in float32 (torch.amax: NaN propagates), then the Hamming
//                  aggregation of post_kernel with one global speaker and the identity map (post_agg.cuh), every output
//                  frame's float64 value written at the chunk's offset in the curve
//   vad_binarize   one warp per (chunk, trial): curve > tau[t], run-length encoded into post_kernel's header
//                  {offset, count, frames, 0} and packed turns (0 << 20 | on << 10 | off), all trials sharing one counter
#include "dg_common.cuh"
#include "post_agg.cuh"

namespace dg {

constexpr unsigned VAD_FULL = 0xffffffffu;
constexpr int VAD_CURVE_THREADS = 64;
constexpr int VAD_BIN_THREADS = 256;

// plan [N][plan_stride] as post_kernel's, without history: chunk c aggregates chunks c - (nb - 1) .. c
__global__ void __launch_bounds__(VAD_CURVE_THREADS)
vad_curve_kernel(const float* __restrict__ seg /*[N][F][K]*/, int F, int K, const int32_t* __restrict__ plan, int plan_stride,
                 const double* __restrict__ hamming, const long long* __restrict__ curve_off /*[N + 1]*/,
                 double* __restrict__ curve) {
  const int c = blockIdx.x;
  const int32_t* pl = plan + (size_t)c * plan_stride;
  const int nb = pl[0], nf = pl[1], first_nf = pl[2], first_lo = pl[3];
  const int nfo = first_nf > 0 ? first_nf : nf;
  double* out = curve + curve_off[c];
  for (int fo = threadIdx.x; fo < nfo; fo += VAD_CURVE_THREADS)
    out[fo] = post_frame(pl, nb, nf, nfo, first_lo, F, hamming, fo, [&](int j, int idx) {
      const float* s = seg + ((size_t)(c - (nb - 1) + j) * F + idx) * K;
      float m = s[0];
      for (int k = 1; k < K; k++) {
        const float x = s[k];
        m = (x > m || isnan(x)) ? x : m;      // a NaN, once taken, is never replaced: x > NaN is false
      }
      return (double)m;
    });
}

// warp (c, t): chunk c of the N, trial t of the T.  Frames 0 .. nfo are read 32 at a time with frame nfo inactive, so that a
// turn still open at the end closes there; a turn's off frame is the lane whose frame is inactive after an active one, its on
// frame the last start before it.
__global__ void __launch_bounds__(VAD_BIN_THREADS)
vad_binarize_kernel(const double* __restrict__ curve, const long long* __restrict__ curve_off /*[N + 1]*/, int N, int T,
                    const double* __restrict__ taus /*[T]*/, int32_t* __restrict__ header /*[T][N][4]*/,
                    uint32_t* __restrict__ turns, int turn_cap, unsigned int* __restrict__ total) {
  const long long w = ((long long)blockIdx.x * VAD_BIN_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)N * T) return;   // the whole warp
  const int t = (int)(w / N), c = (int)(w - (long long)t * N);
  const double tau = taus[t];
  const double* v = curve + curve_off[c];
  const int nfo = (int)(curve_off[c + 1] - curve_off[c]);
  const unsigned below = (1u << lane) - 1u;
  // pass 1: the number of turns
  int n = 0;
  unsigned carry = 0;   // frame f0 - 1 active
  for (int f0 = 0; f0 <= nfo; f0 += 32) {
    const int f = f0 + lane;
    const unsigned act = __ballot_sync(VAD_FULL, f < nfo && v[f] > tau);
    n += __popc(act & ~((act << 1) | carry));
    carry = act >> 31;
  }
  unsigned base = 0;
  if (lane == 0 && n > 0) base = atomicAdd(total, (unsigned)n);
  base = __shfl_sync(VAD_FULL, base, 0);
  if (lane == 0) {
    int32_t* hd = header + ((size_t)t * N + c) * 4;
    hd[0] = (int32_t)base;
    hd[1] = n;
    hd[2] = nfo;
    hd[3] = 0;
  }
  if (n == 0) return;
  // pass 2: the turns, in time order
  int done = 0, on = 0;
  carry = 0;
  for (int f0 = 0; f0 <= nfo; f0 += 32) {
    const int f = f0 + lane;
    const unsigned act = __ballot_sync(VAD_FULL, f < nfo && v[f] > tau);
    const unsigned prev = (act << 1) | carry;
    const unsigned starts = act & ~prev, ends = ~act & prev;
    if ((ends >> lane) & 1u) {
      const unsigned s = starts & below;
      const int my_on = s ? f0 + 31 - __clz(s) : on;
      const size_t o = (size_t)base + done + __popc(ends & below);
      if (o < (size_t)turn_cap) turns[o] = ((uint32_t)my_on << 10) | (uint32_t)f;
    }
    done += __popc(ends);
    if (starts) on = f0 + 31 - __clz(starts);
    carry = act >> 31;
  }
}

int launch_vad_curve(const float* seg, int N, int F, int K, const int32_t* plan, int plan_stride, const double* hamming,
                     const long long* curve_off, double* curve, cudaStream_t st) {
  ProfScope _ps("vad_curve", st);
  vad_curve_kernel<<<N, VAD_CURVE_THREADS, 0, st>>>(seg, F, K, plan, plan_stride, hamming, curve_off, curve);
  DG_LAUNCHED();
  return 0;
}

int launch_vad_binarize(const double* curve, const long long* curve_off, int N, int T, const double* taus, int32_t* header,
                        uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st) {
  ProfScope _ps("vad_binarize", st);
  const unsigned blocks = (unsigned)(((long long)N * T * 32 + VAD_BIN_THREADS - 1) / VAD_BIN_THREADS);
  vad_binarize_kernel<<<blocks, VAD_BIN_THREADS, 0, st>>>(curve, curve_off, N, T, taus, header, turns, turn_cap, total);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

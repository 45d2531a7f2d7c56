// Voice activity detection sweep on the device: the reference tunes VoiceActivityDetection's only hyper-parameter, tau_active,
// by running the whole pipeline once per trial (Optimizer.objective -> Benchmark, reference src/diart/optim.py:98-122).  The
// threshold is read by Binarize alone (blocks/vad.py:150-180), so here the speech curve -- the max over the local speakers
// (vad.py:145-148) aggregated over the `latency / step` most recent chunks -- is computed once per dataset and every trial
// only compares it with its own threshold.
//
//   vad_curve      one CTA per chunk: max over the K local speakers in float32 (torch.amax: NaN propagates), then the Hamming
//                  aggregation of the post-path with one global speaker and the identity map (post_agg.cuh), every output
//                  frame's float64 value written at the chunk's offset in the curve
//   vad_binarize   one warp per (chunk, trial): curve > tau[t], run-length encoded into the post-path's header
//                  {offset, count, frames, 0} and packed turns (0 << 20 | on << 10 | off), all trials sharing one counter
//
// Many live VAD streams (dg_multi in VAD mode) use the same two bodies, per tick and per stream:
//
//   vad_slots          one CTA per chunk of the tick: its speech curve (max over the local speakers of this tick's scores or
//                      the slot's history of max curves, aggregated as vad_curve aggregates) compared with tau, run-length
//                      encoded as vad_binarize encodes it
//   vad_slots_history  the last nw - 1 max curves of every slot of the tick into the other copy of its history
#include "dg_common.cuh"
#include "post_agg.cuh"

namespace dg {

constexpr unsigned VAD_FULL = 0xffffffffu;
constexpr int VAD_CURVE_THREADS = 64;
constexpr int VAD_BIN_THREADS = 256;
constexpr int VAD_SLOTS_THREADS = 64;

// plan [Nv][plan_stride] as the post-path's, without history: chunk c is real chunk vchunk[c] of seg (vchunk null: chunk c),
// and buffer j of its plan row the real chunk vchunk[c] - (nb - 1) + j
__global__ void __launch_bounds__(VAD_CURVE_THREADS)
vad_curve_virtual_kernel(const float* __restrict__ seg /*[N][F][K]*/, const int32_t* __restrict__ vchunk, int F, int K,
                         const int32_t* __restrict__ plan, int plan_stride, const double* __restrict__ hamming,
                         const long long* __restrict__ curve_off /*[Nv + 1]*/, double* __restrict__ curve) {
  const int c = blockIdx.x;
  const int32_t* pl = plan + (size_t)c * plan_stride;
  const int nb = pl[0], nf = pl[1], first_nf = pl[2], first_lo = pl[3];
  const int nfo = first_nf > 0 ? first_nf : nf;
  const int r0 = (vchunk ? vchunk[c] : c) - (nb - 1);
  double* out = curve + curve_off[c];
  for (int fo = threadIdx.x; fo < nfo; fo += VAD_CURVE_THREADS)
    out[fo] = post_frame(pl, nb, nf, nfo, first_lo, F, hamming, fo, [&](int j, int idx) {
      return (double)speaker_max(seg + ((size_t)(r0 + j) * F + idx) * K, K);
    });
}

// One warp run-length encodes the frames 0 .. nfo - 1 of a chunk into its header row hd {offset, count, frames, 0} and its
// packed turns (0 << 20 | on << 10 | off), placed with one atomicAdd on `total`.  word(f0) is the ballot of the active frames
// f0 .. f0 + 31 (none at or beyond nfo), read 32 at a time up to frame nfo, which is inactive, so that a turn still open at
// the end closes there; a turn's off frame is the lane whose frame is inactive after an active one, its on frame the last
// start before it.
template <class Word>
__device__ __forceinline__ void warp_turns(int nfo, Word word, int32_t* __restrict__ hd, uint32_t* __restrict__ turns,
                                           int turn_cap, unsigned int* __restrict__ total) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  // pass 1: the number of turns
  int n = 0;
  unsigned carry = 0;   // frame f0 - 1 active
  for (int f0 = 0; f0 <= nfo; f0 += 32) {
    const unsigned act = word(f0);
    n += __popc(act & ~((act << 1) | carry));
    carry = act >> 31;
  }
  unsigned base = 0;
  if (lane == 0 && n > 0) base = atomicAdd(total, (unsigned)n);
  base = __shfl_sync(VAD_FULL, base, 0);
  if (lane == 0) {
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
    const unsigned act = word(f0);
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

// warp (c, t): chunk c of the N, trial t of the T
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
  warp_turns(nfo, [&](int f0) {
    const int f = f0 + lane;
    return __ballot_sync(VAD_FULL, f < nfo && v[f] > tau);
  }, header + ((size_t)t * N + c) * 4, turns, turn_cap, total);
}

// Many live streams (dg_multi in VAD mode), one CTA per chunk of the tick: chunk c is window rows[c].y of slot entry
// act[rows[c].x], as in post_slots_kernel (post.cu).  Buffer j of its plan row is a row of this tick's scores seg [B][F][K],
// max over the K local speakers, or an entry of the slot's history hist_vad [2][slots][nw - 1][F] (copy `cur`, n_hist entries,
// oldest first), which holds such max curves already.  Each output frame is post_chunk's value with one speaker and the
// identity map -- the same float64 expression in the same order -- compared with `> tau`, tau = params[3 * rows[c].x] (the
// stream's tau_active); the two warps ballot 32 frames at a time into `bits`, then warp 0 run-length encodes them.  nw is the
// largest latency / step of any slot (the history stride); the plan row's nb <= ts.nw.
__global__ void __launch_bounds__(VAD_SLOTS_THREADS)
vad_slots_kernel(const float* __restrict__ seg, const float* __restrict__ hist_vad, const TickSlot* __restrict__ act,
                 const int2* __restrict__ rows, int slots, int F, int K, int nw, const int32_t* __restrict__ plan,
                 int plan_stride, const double* __restrict__ hamming, const double* __restrict__ params,
                 int32_t* __restrict__ header, uint32_t* __restrict__ turns, int turn_cap, unsigned int* __restrict__ total) {
  __shared__ unsigned bits[(1024 + 32) / 32];   // frames 0 .. nfo <= F + 1 <= 1024
  const int c = blockIdx.x;
  const int2 r = rows[c];
  const TickSlot ts = act[r.x];
  const double tau = params[(size_t)r.x * 3];
  const int32_t* pl = plan + (size_t)c * plan_stride;
  const int nb = pl[0], nf = pl[1], first_nf = pl[2], first_lo = pl[3];
  const int nfo = first_nf > 0 ? first_nf : nf;
  const size_t h0 = ((size_t)ts.cur * slots + ts.slot) * (nw - 1) + ts.n_hist;   // one past the slot's newest history entry
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int q = warp; q * 32 <= nfo; q += VAD_SLOTS_THREADS / 32) {
    const int fo = q * 32 + lane;
    bool on = false;
    if (fo < nfo)
      on = post_frame(pl, nb, nf, nfo, first_lo, F, hamming, fo, [&](int j, int idx) {
             const int v = r.y - (nb - 1) + j;     // virtual chunk of the slot; v < 0 lives in its history
             return (double)(v >= 0 ? speaker_max(seg + ((size_t)(ts.row0 + v) * F + idx) * K, K)
                                    : hist_vad[(h0 + v) * F + idx]);
           }) > tau;
    const unsigned word = __ballot_sync(VAD_FULL, on);
    if (lane == 0) bits[q] = word;
  }
  __syncthreads();
  if (warp == 0) warp_turns(nfo, [&](int f0) { return bits[f0 >> 5]; }, header + (size_t)c * 4, turns, turn_cap, total);
}

// History update of the VAD slots: CTA (a, i) writes entry i of slot act[a]'s other copy, the last keep = min(ts.nw - 1,
// n_hist + n) chunks of (its history + its n chunks of this tick) as max curves [F], at the stride of the largest slot's
// nw - 1.  The host then flips `cur` and sets n_hist = keep.
__global__ void __launch_bounds__(256)
vad_slots_history_kernel(const float* __restrict__ seg, float* hist_vad, const TickSlot* __restrict__ act, int slots, int F,
                         int K, int nw) {
  const TickSlot ts = act[blockIdx.x];
  const int i = blockIdx.y;
  const int keep = min(ts.nw - 1, ts.n_hist + ts.n);
  if (i >= keep) return;
  const int v = ts.n - keep + i;                    // virtual chunk: v >= 0 is this tick's, v < 0 the history's
  const size_t src = ((size_t)ts.cur * slots + ts.slot) * (nw - 1) + ts.n_hist;
  const size_t dst = ((size_t)(ts.cur ^ 1) * slots + ts.slot) * (nw - 1) + i;
  for (int f = threadIdx.x; f < F; f += blockDim.x)
    hist_vad[dst * F + f] = v >= 0 ? speaker_max(seg + ((size_t)(ts.row0 + v) * F + f) * K, K) : hist_vad[(src + v) * F + f];
}

int launch_vad_curve_virtual(const float* seg, const int32_t* vchunk, int Nv, int F, int K, const int32_t* plan, int plan_stride,
                             const double* hamming, const long long* curve_off, double* curve, cudaStream_t st) {
  ProfScope _ps("vad_curve", st);
  vad_curve_virtual_kernel<<<Nv, VAD_CURVE_THREADS, 0, st>>>(seg, vchunk, F, K, plan, plan_stride, hamming, curve_off, curve);
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

int launch_vad_slots(const float* seg, const float* hist_vad, const TickSlot* act, const int2* rows, int slots, int B, int F,
                     int K, int nw, const int32_t* plan, int plan_stride, const double* hamming, const double* params,
                     int32_t* header, uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st) {
  ProfScope _ps("vad_slots", st);
  if (F > 1023) {
    set_error("vad_slots: at most 1023 frames");
    return -1;
  }
  vad_slots_kernel<<<B, VAD_SLOTS_THREADS, 0, st>>>(seg, hist_vad, act, rows, slots, F, K, nw, plan, plan_stride, hamming,
                                                    params, header, turns, turn_cap, total);
  DG_LAUNCHED();
  return 0;
}

int launch_vad_slots_history(const float* seg, float* hist_vad, const TickSlot* act, int n_act, int slots, int F, int K, int nw,
                             cudaStream_t st) {
  ProfScope _ps("vad_slots_history", st);
  if (n_act < 1 || nw < 2) return 0;
  vad_slots_history_kernel<<<dim3(n_act, nw - 1), 256, 0, st>>>(seg, hist_vad, act, slots, F, K, nw);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

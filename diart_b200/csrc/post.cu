// Post-path of SpeakerDiarization.__call__ on the device (reference src/diart/blocks/diarization.py:205-232):
//
//   SpeakerMap.apply           permuted[:, g] = seg[:, k] for every mapped local speaker      mapping.py:341-360
//   DelayedAggregation         Hamming-weighted average of the `latency / step` most recent permuted buffers over the
//                              region that ends `latency` before the newest buffer's end        aggregation.py:73-92,120-218
//                              (+ the first-buffer prepend rule, aggregation.py:188-212)
//   Binarize                   scores > tau, run-length encoded into (speaker, on, off) turns    blocks/utils.py:11-59
//
// The frame ranges (`SlidingWindow.crop(mode="loose", fixed=...)`, pyannote.core) are float64 index arithmetic on chunk
// start times that only the host knows; the host passes them per chunk as a small integer plan (diart_b200/blocks/post.py),
// the device does everything that touches scores.  Arithmetic follows numpy statement by statement in float64 WITHOUT
// fused multiply-add -- np.sum(ham * val, axis=0) / np.sum(ham, axis=0) adds the buffers in order -- so the thresholded
// result is bit-identical to the reference's, not merely close.
//
// One CTA per chunk.  Output: per chunk {offset, count, frames} and a packed turn list (speaker << 20 | on << 10 | off),
// each chunk's turns contiguous, ordered by speaker then time (the order Binarize emits them).
//
// Two kernels run that body: post_slots_kernel over the chunks of live streams, each with its history (dg_post is one such
// stream, dg_multi many), and post_virtual_kernel over the chunks of a sweep, without history, with a second grid dimension
// for independent states (trials) over the same scores.  Every plan row they read has passed check_plan_row (api_post.cu).
#include "dg_common.cuh"
#include "post_agg.cuh"

namespace dg {

constexpr int POST_THREADS = 256;

// plan row (int32): [0] nb buffers aggregated, [1] nf frames of the region crop, [2] first_nf (> 0: first buffer of a
// stream, output = crop of [0, region.end) with its last nf frames replaced), [3] first_lo, [4 ..] lo of each buffer
//
// The body of the post-path for chunk c (one CTA): buf_seg(j) / buf_map(j) are the scores [F][K] and map [K] of its buffer j,
// oldest first; writes header row c and the chunk's turns.
template <class BufSeg, class BufMap>
__device__ __forceinline__ void post_chunk(const int32_t* __restrict__ pl, int c, int nb, int nf, int first_nf, int first_lo,
                                           int F, int K, int M, int nw, const double* __restrict__ hamming, double tau,
                                           int32_t* __restrict__ header, uint32_t* __restrict__ turns, int turn_cap,
                                           unsigned int* __restrict__ total, BufSeg buf_seg, BufMap buf_map) {
  extern __shared__ unsigned char sm_raw[];
  const int nfo = first_nf > 0 ? first_nf : nf;
  signed char* inv = reinterpret_cast<signed char*>(sm_raw);           // [nb][M]: local speaker of global g, or -1
  unsigned char* act = sm_raw + ((nw * M + 15) & ~15);                    // [nfo][M]
  __shared__ int cnt[64], off[65];
  __shared__ unsigned int base_s;

  for (int i = threadIdx.x; i < nb * M; i += POST_THREADS) inv[i] = -1;
  __syncthreads();
  if (threadIdx.x < nb) {
    const int32_t* mp = buf_map(threadIdx.x);
    for (int k = 0; k < K; k++) {          // ascending k: a later local speaker overwrites (as the reference's loop would)
      const int g = mp[k];
      if (g >= 0 && g < M) inv[threadIdx.x * M + g] = (signed char)k;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nfo * M; i += POST_THREADS) {
    const int fo = i / M, g = i - fo * M;
    const double v = post_frame(pl, nb, nf, nfo, first_lo, F, hamming, fo, [&](int j, int idx) {
      const int k = inv[j * M + g];
      return k >= 0 ? (double)buf_seg(j)[(size_t)idx * K + k] : 0.0;
    });
    act[i] = v > tau ? 1 : 0;
  }
  __syncthreads();
  // run-length encode per speaker (thread g), two passes around a prefix sum
  const int g = threadIdx.x;
  int n = 0;
  if (g < M) {
    int prev = 0;
    for (int f = 0; f < nfo; f++) {
      const int a = act[f * M + g];
      n += (a && !prev);
      prev = a;
    }
    cnt[g] = n;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int i = 0; i < M; i++) {
      off[i] = s;
      s += cnt[i];
    }
    off[M] = s;
    base_s = atomicAdd(total, (unsigned int)s);
    header[c * 4 + 0] = (int32_t)base_s;
    header[c * 4 + 1] = s;
    header[c * 4 + 2] = nfo;
    header[c * 4 + 3] = 0;
  }
  __syncthreads();
  if (g < M && n > 0) {
    size_t o = (size_t)base_s + off[g];
    int prev = 0, on = 0;
    for (int f = 0; f <= nfo; f++) {
      const int a = f < nfo ? act[f * M + g] : 0;
      if (a && !prev) on = f;
      if (!a && prev) {
        if (o < (size_t)turn_cap) turns[o] = ((uint32_t)g << 20) | ((uint32_t)on << 10) | (uint32_t)f;
        o++;
      }
      prev = a;
    }
  }
}

// The sweeps (dg_sweep_*): CTA (c, t) is virtual chunk c of the gridDim.x and trial t.  The scores seg [N][F][K] and maps
// [T][N][K] are over the N real chunks; virtual chunk c is real chunk vchunk[c] (vchunk null: chunk c), and buffer j of its
// plan row the real chunk vchunk[c] - (nb - 1) + j, inside the chunk's own file.  Header [T][gridDim.x][4]; trial t
// thresholds at taus[t].  A virtual chunk's turns are the bits of the real chunk at its latency.
__global__ void __launch_bounds__(POST_THREADS)
post_virtual_kernel(const float* __restrict__ seg, const int32_t* __restrict__ map, int N, const int32_t* __restrict__ vchunk,
                    int F, int K, int M, int nw, const int32_t* __restrict__ plan, int plan_stride,
                    const double* __restrict__ hamming, const double* __restrict__ taus, int32_t* __restrict__ header,
                    uint32_t* __restrict__ turns, int turn_cap, unsigned int* __restrict__ total) {
  const int c = blockIdx.x;
  map += (size_t)blockIdx.y * N * K;
  header += (size_t)blockIdx.y * gridDim.x * 4;
  const double tau = taus[blockIdx.y];
  const int32_t* pl = plan + (size_t)c * plan_stride;
  const int nb = pl[0], nf = pl[1], first_nf = pl[2], first_lo = pl[3];
  const int r0 = (vchunk ? vchunk[c] : c) - (nb - 1);     // real chunk of buffer 0
  auto buf_seg = [&](int j) -> const float* { return seg + (size_t)(r0 + j) * F * K; };
  auto buf_map = [&](int j) -> const int32_t* { return map + (size_t)(r0 + j) * K; };
  post_chunk(pl, c, nb, nf, first_nf, first_lo, F, K, M, nw, hamming, tau, header, turns, turn_cap, total, buf_seg, buf_map);
}

// Live streams in one batch (dg_multi; dg_post is one stream in slot 0): the B chunks are grouped by stream slot.  Chunk c
// is window rows[c].y of this batch's slot entry act[rows[c].x] (TickSlot, dg_common.cuh), whose chunks start at batch row
// row0.  Each slot has its own history of up to ts.nw - 1 <= nw - 1 chunks: hist_seg [2][slots][nw - 1][F][K] and hist_map
// [2][slots][nw - 1][K] (two copies, `cur` is the current one), of which the first n_hist entries hold the last chunks seen,
// oldest first.  nw is the largest of the slots' (it sizes the history and the shared memory); a chunk aggregates the
// nb <= ts.nw buffers of its plan row and compares with its entry's tau, params[3 * rows[c].x], the value a dedicated
// post-path at that stream's tau_active compares with.
__global__ void __launch_bounds__(POST_THREADS)
post_slots_kernel(const float* __restrict__ seg, const int32_t* __restrict__ map, const float* __restrict__ hist_seg,
                  const int32_t* __restrict__ hist_map, const TickSlot* __restrict__ act, const int2* __restrict__ rows,
                  int slots, int F, int K, int M, int nw, const int32_t* __restrict__ plan, int plan_stride,
                  const double* __restrict__ hamming, const double* __restrict__ params, int32_t* __restrict__ header,
                  uint32_t* __restrict__ turns, int turn_cap, unsigned int* __restrict__ total) {
  const int c = blockIdx.x;
  const int2 r = rows[c];
  const TickSlot ts = act[r.x];
  const double tau = params[(size_t)r.x * 3];
  const int32_t* pl = plan + (size_t)c * plan_stride;
  const int nb = pl[0], nf = pl[1], first_nf = pl[2], first_lo = pl[3];
  const size_t h0 = ((size_t)ts.cur * slots + ts.slot) * (nw - 1) + ts.n_hist;   // one past the slot's newest history entry
  // buffer j of this chunk = virtual chunk v of its slot; v < 0 lives in the slot's history
  auto buf_seg = [&](int j) -> const float* {
    const int v = r.y - (nb - 1) + j;
    return v >= 0 ? seg + (size_t)(ts.row0 + v) * F * K : hist_seg + (h0 + v) * F * K;
  };
  auto buf_map = [&](int j) -> const int32_t* {
    const int v = r.y - (nb - 1) + j;
    return v >= 0 ? map + (size_t)(ts.row0 + v) * K : hist_map + (h0 + v) * K;
  };
  post_chunk(pl, c, nb, nf, first_nf, first_lo, F, K, M, nw, hamming, tau, header, turns, turn_cap, total, buf_seg, buf_map);
}

// History update of the slots of a dg_multi batch: CTA (a, i) writes entry i of slot act[a]'s other history copy, the last
// keep = min(ts.nw - 1, n_hist + n) chunks of (its history + its n chunks of this batch); the stride of the entries is the
// largest slot's nw - 1.  The host then flips `cur` and sets n_hist = keep.
__global__ void __launch_bounds__(256)
post_slots_history_kernel(const float* __restrict__ seg, const int32_t* __restrict__ map, float* __restrict__ hist_seg,
                          int32_t* __restrict__ hist_map, const TickSlot* __restrict__ act, int slots, int FK, int K, int nw) {
  const TickSlot ts = act[blockIdx.x];
  const int i = blockIdx.y;
  const int keep = min(ts.nw - 1, ts.n_hist + ts.n);
  if (i >= keep) return;
  const int v = ts.n - keep + i;                    // virtual chunk: v >= 0 is this batch's, v < 0 the history's
  const size_t src = ((size_t)ts.cur * slots + ts.slot) * (nw - 1) + ts.n_hist;
  const size_t dst = ((size_t)(ts.cur ^ 1) * slots + ts.slot) * (nw - 1) + i;
  const float* s = v >= 0 ? seg + (size_t)(ts.row0 + v) * FK : hist_seg + (src + v) * FK;
  const int32_t* m = v >= 0 ? map + (size_t)(ts.row0 + v) * K : hist_map + (src + v) * K;
  for (int e = threadIdx.x; e < FK; e += blockDim.x) hist_seg[dst * FK + e] = s[e];
  for (int e = threadIdx.x; e < K; e += blockDim.x) hist_map[dst * K + e] = m[e];
}

// The launch set-up of both post kernels: the limit checks and post_chunk's dynamic shared memory, inv [nw][M] then act
// [F + 1][M] (the first chunk of a stream or file emits the crop of [0, region end), up to F + 1 frames), with the opt-in
// above 48 KB once per device (`attr_done`: the launcher's flags).
template <class Kern>
static int post_setup(const char* who, Kern* kern, bool* attr_done, int F, int K, int M, int nw, size_t* smem) {
  if (M > 64 || F > 1023 || K > 127) {
    set_error(std::string(who) + ": at most 64 global speakers, 1023 frames");
    return -1;
  }
  *smem = ((size_t)(nw * M + 15) & ~(size_t)15) + (size_t)(F + 1) * M;
  if (*smem > 200 * 1024) {
    set_error(std::string(who) + ": latency / step too large for the shared-memory plan");
    return -1;
  }
  if (*smem > 48 * 1024 && first_use_on_device(attr_done))
    DG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  return 0;
}

int launch_post_virtual(const float* seg, const int32_t* map, int N, const int32_t* vchunk, int Nv, int F, int K, int M, int nw,
                        const int32_t* plan, int plan_stride, const double* hamming, const double* taus, int T,
                        int32_t* header, uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st) {
  ProfScope _ps("post_virtual", st);
  if (T < 1 || T > 65535 || !taus || Nv < 1) {
    set_error("post_virtual: 1 <= states <= 65535 with per-state thresholds, at least one chunk");
    return -1;
  }
  static bool attr_done[64] = {};
  size_t smem = 0;
  int rc;
  if ((rc = post_setup("post_virtual", post_virtual_kernel, attr_done, F, K, M, nw, &smem))) return rc;
  post_virtual_kernel<<<dim3(Nv, T), POST_THREADS, smem, st>>>(seg, map, N, vchunk, F, K, M, nw, plan, plan_stride, hamming,
                                                               taus, header, turns, turn_cap, total);
  DG_LAUNCHED();
  return 0;
}

// ---- device-side rearrange_audio_stream (reference src/diart/operators.py:44-100): windows of a circular sample ring
// window b = samples [r0 + b*hop, r0 + b*hop + S) of the stream, ring index = absolute sample index mod C (C % 4 == 0,
// r0 % 4 == 0, hop % 4 == 0, S % 4 == 0: 16-byte accesses never straddle the wrap)
__global__ void __launch_bounds__(256) expand_windows_kernel(const float* __restrict__ ring, long long r0, int C, int hop, int S,
                                                             float* __restrict__ wav) {
  const int b = blockIdx.y;
  const long long base = r0 + (long long)b * hop;
  float4* dst = reinterpret_cast<float4*>(wav + (size_t)b * S);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (S >> 2); i += gridDim.x * blockDim.x) {
    const int idx = (int)((base + 4LL * i) % C);
    dst[i] = *reinterpret_cast<const float4*>(ring + idx);
  }
}

int launch_expand_windows(const float* ring, long long r0, int C, int hop, int S, int B, float* wav, cudaStream_t st) {
  ProfScope _ps("expand_windows", st);
  dim3 grid(8, B);
  expand_windows_kernel<<<grid, 256, 0, st>>>(ring, r0, C, hop, S, wav);
  DG_LAUNCHED();
  return 0;
}

// ---- the rings of many streams (dg_multi): slot s owns rings [s][C]; absolute sample t of a slot lives at index t mod C.
// Piece p of the staging buffer (one upload of every stream's new samples) goes to its slot's ring; CTA b takes pieces b,
// b + gridDim.x, ..., so any number of pieces fits one launch.
__global__ void __launch_bounds__(256) ring_scatter_kernel(const float* __restrict__ staged, const RingPiece* __restrict__ pieces,
                                                           int n_pieces, int C, float* __restrict__ rings) {
  for (int q = blockIdx.x; q < n_pieces; q += gridDim.x) {
    const RingPiece p = pieces[q];
    float* ring = rings + (size_t)p.slot * C;
    for (int i = threadIdx.x; i < p.n; i += blockDim.x) ring[(p.dst + i) % C] = staged[p.src + i];
  }
}

// entry b of rows = samples [start[b], start[b] + S) of the ring of slot act[rows[b].x].slot, to batch row act[..].row0 +
// rows[b].y (C, start, S multiples of 4: 16-byte accesses never straddle the wrap)
__global__ void __launch_bounds__(256) ring_gather_kernel(const float* __restrict__ rings, int C, const TickSlot* __restrict__ act,
                                                          const int2* __restrict__ rows, const long long* __restrict__ start,
                                                          int S, float* __restrict__ wav) {
  const int b = blockIdx.y;
  const int2 r = rows[b];
  const TickSlot& ts = act[r.x];
  const float* ring = rings + (size_t)ts.slot * C;
  const long long base = start[b];
  float4* dst = reinterpret_cast<float4*>(wav + (size_t)(ts.row0 + r.y) * S);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (S >> 2); i += gridDim.x * blockDim.x) {
    const int idx = (int)((base + 4LL * i) % C);
    dst[i] = *reinterpret_cast<const float4*>(ring + idx);
  }
}

int launch_ring_scatter(const float* staged, const RingPiece* pieces, int n_pieces, int C, float* rings, cudaStream_t st) {
  ProfScope _ps("ring_scatter", st);
  if (n_pieces < 1) return 0;
  ring_scatter_kernel<<<n_pieces < 4096 ? n_pieces : 4096, 256, 0, st>>>(staged, pieces, n_pieces, C, rings);
  DG_LAUNCHED();
  return 0;
}

int launch_ring_gather(const float* rings, int C, const TickSlot* act, const int2* rows, const long long* start, int S, int B,
                       float* wav, cudaStream_t st) {
  ProfScope _ps("ring_gather", st);
  if (B > 65535) {
    set_error("ring_gather: at most 65535 windows per batch");
    return -1;
  }
  ring_gather_kernel<<<dim3(8, B), 256, 0, st>>>(rings, C, act, rows, start, S, wav);
  DG_LAUNCHED();
  return 0;
}

int launch_post_slots(const float* seg, const int32_t* map, const float* hist_seg, const int32_t* hist_map,
                      const TickSlot* act, const int2* rows, int slots, int B, int F, int K, int M, int nw,
                      const int32_t* plan, int plan_stride, const double* hamming, const double* params, int32_t* header,
                      uint32_t* turns, int turn_cap, unsigned int* total, cudaStream_t st) {
  ProfScope _ps("post_slots", st);
  static bool attr_done[64] = {};
  size_t smem = 0;
  int rc;
  if ((rc = post_setup("post_slots", post_slots_kernel, attr_done, F, K, M, nw, &smem))) return rc;
  post_slots_kernel<<<B, POST_THREADS, smem, st>>>(seg, map, hist_seg, hist_map, act, rows, slots, F, K, M, nw, plan,
                                                   plan_stride, hamming, params, header, turns, turn_cap, total);
  DG_LAUNCHED();
  return 0;
}

int launch_post_slots_history(const float* seg, const int32_t* map, float* hist_seg, int32_t* hist_map, const TickSlot* act,
                              int n_act, int slots, int F, int K, int nw, cudaStream_t st) {
  ProfScope _ps("post_slots_history", st);
  if (n_act < 1 || nw < 2) return 0;
  post_slots_history_kernel<<<dim3(n_act, nw - 1), 256, 0, st>>>(seg, map, hist_seg, hist_map, act, slots, F * K, K, nw);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

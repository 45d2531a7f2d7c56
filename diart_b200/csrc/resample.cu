// Polyphase sinc resampling of audio windows (torchaudio.functional.resample with its defaults, which the reference's
// blocks.Resample applies to every window of a source whose rate differs from the pipeline's; reference
// src/diart/blocks/utils.py:62-89, src/diart/inference.py:101-123).
//
// With o / n the reduced rate ratio, w the filter half-width and W the [n][T = 2w + o] float32 tap table built on the host:
//   y[r n + p] = sum_k x[r o + k - w] W[p][k],   x = 0 outside the window,   output length ceil(n L / o).
// Every output is ONE float32 accumulator updated in tap order k = 0 .. T-1 with fmaf, zeros standing in for the padding,
// whichever kernel computes it.  That makes the per-window form, the stream form (outputs of the batch's unique source samples,
// shared by the overlapping windows) and the crops bit-identical to each other.
#include "dg_common.cuh"

#include <algorithm>

namespace dg {

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr size_t RS_SMEM_MAX = 200 * 1024;

// launch shape: each thread accumulates QF frames (lane + 32 f) x QP phases; a block covers FG groups of 32 QF frames and
// every phase, with the source samples of its frames staged in shared memory (the tap table is read through L1: all lanes of
// a warp read the same tap)
struct RsPlan {
  int qf, qp, fg, tile_frames;
  size_t smem;
};

RsPlan rs_plan(const RsGeom& g) {
  RsPlan p;
  p.qp = g.n == 1 ? 1 : 2;
  p.qf = g.n == 1 ? 4 : 2;
  const int npairs = (g.n + p.qp - 1) / p.qp;
  auto smem = [&](int fg) { return ((size_t)(fg * 32 * p.qf - 1) * g.o + g.T) * 4; };
  p.fg = std::max(1, std::min(8, (RS_WARPS + npairs - 1) / npairs));
  while (p.fg > 1 && smem(p.fg) > RS_SMEM_MAX) p.fg--;
  p.tile_frames = p.fg * 32 * p.qf;
  p.smem = smem(p.fg);
  return p;
}

__device__ __forceinline__ RsItem rs_item(const RsJob& j, int b) {
  if (j.items) return j.items[b];
  RsItem it = j.base;
  it.start += (long long)b * j.start_step;
  it.out_off += (long long)b * j.out_step;
  return it;
}

// The tap loop of a tile: warps take (frame group, phase pair) items; a lane accumulates frames r0 + grp 32 QF + lane + 32 f of
// phases p0 .. p0 + QP - 1 from the staged source samples xs (xs[0] = tap 0 of frame r0) and hands each result to
// store(frame r, p0, q, value) (phase p0 + q < n).  The caller synchronises after staging xs.
template <int QF, int QP, class Store>
__device__ __forceinline__ void rs_tile_taps(const float* xs, const float* W, int o, int n, int T, int fg,
                                             long long r0, Store store) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int npairs = (n + QP - 1) / QP;
  for (int wi = warp; wi < fg * npairs; wi += RS_WARPS) {
    const int grp = wi / npairs, p0 = (wi % npairs) * QP;
    const float* wr[QP];
#pragma unroll
    for (int q = 0; q < QP; ++q) wr[q] = W + (size_t)min(p0 + q, n - 1) * T;
    const float* xr = xs + (size_t)(grp * 32 * QF + lane) * o;
    float acc[QF][QP];
#pragma unroll
    for (int f = 0; f < QF; ++f)
#pragma unroll
      for (int q = 0; q < QP; ++q) acc[f][q] = 0.f;
    for (int k = 0; k < T; ++k) {
      float wk[QP];
#pragma unroll
      for (int q = 0; q < QP; ++q) wk[q] = __ldg(wr[q] + k);
#pragma unroll
      for (int f = 0; f < QF; ++f) {
        const float xv = xr[(size_t)f * 32 * o + k];
#pragma unroll
        for (int q = 0; q < QP; ++q) acc[f][q] = __fmaf_rn(xv, wk[q], acc[f][q]);
      }
    }
#pragma unroll
    for (int f = 0; f < QF; ++f) {
      const long long r = r0 + grp * 32 * QF + lane + 32 * f;
#pragma unroll
      for (int q = 0; q < QP; ++q) store(r, p0, q, acc[f][q]);
    }
  }
}

template <int QF, int QP>
__global__ void __launch_bounds__(RS_THREADS) resample_tile_kernel(RsJob j, int fg) {
  extern __shared__ float xs[];
  const RsItem it = rs_item(j, blockIdx.y);
  const int o = j.g.o, n = j.g.n, T = j.g.T;
  const long long j_end = it.j_lo + it.j_cnt;
  const long long r0 = it.j_lo / n + (long long)blockIdx.x * fg * 32 * QF;
  if (r0 * n >= j_end) return;
  // source samples [t0, t0 + span) of the item, zero outside [0, len)
  const int span = (fg * 32 * QF - 1) * o + T;
  const long long t0 = r0 * o - j.g.w;
  if (j.C) {
    long long a0 = (it.start + t0) % j.C;
    if (a0 < 0) a0 += j.C;
    for (int i = threadIdx.x; i < span; i += RS_THREADS) {
      const long long t = t0 + i;
      long long a = a0 + i;
      while (a >= j.C) a -= j.C;
      xs[i] = (t >= 0 && t < it.len) ? __ldg(j.x + a) : 0.f;
    }
  } else {
    for (int i = threadIdx.x; i < span; i += RS_THREADS) {
      const long long t = t0 + i;
      xs[i] = (t >= 0 && t < it.len) ? __ldg(j.x + it.start + t) : 0.f;
    }
  }
  __syncthreads();
  float* out = j.out + it.out_off;
  rs_tile_taps<QF, QP>(xs, j.W, o, n, T, fg, r0, [&](long long r, int p0, int q, float v) {
    const long long jj = r * n + p0 + q;
    if (p0 + q < n && jj >= it.j_lo && jj < j_end) out[jj - it.j_lo] = v;
  });
}

// dg_multi: frames [first, first + count) of the stream in ring `slot` (stride C, absolute sample t at t mod C), written to
// frame R mod Q of that slot's 16 kHz ring (stride Y floats, frame R = outputs [R n, R n + n)).  Every tap of those frames is
// a pushed sample of the stream, so no padding enters; the tile's frames past the item read whatever the ring holds and are
// not stored.
template <int QF, int QP>
__global__ void __launch_bounds__(RS_THREADS) resample_frames_kernel(const float* __restrict__ rings, long long C,
                                                                     const RsFrames* __restrict__ items,
                                                                     const float* __restrict__ W, RsGeom g,
                                                                     float* __restrict__ yrings, long long Y, long long Q,
                                                                     int fg) {
  extern __shared__ float xs[];
  const RsFrames it = items[blockIdx.y];
  const int o = g.o, n = g.n, T = g.T;
  const long long r_end = it.first + it.count;
  const long long r0 = it.first + (long long)blockIdx.x * fg * 32 * QF;
  if (r0 >= r_end) return;
  const int span = (fg * 32 * QF - 1) * o + T;
  const float* x = rings + (size_t)it.slot * C;
  const long long a0 = (r0 * o - g.w) % C;   // r0 o >= w: the first tap is a pushed sample
  for (int i = threadIdx.x; i < span; i += RS_THREADS) {
    long long a = a0 + i;
    while (a >= C) a -= C;
    xs[i] = __ldg(x + a);
  }
  __syncthreads();
  float* y = yrings + (size_t)it.slot * Y;
  rs_tile_taps<QF, QP>(xs, W, o, n, T, fg, r0, [&](long long r, int p0, int q, float v) {
    if (p0 + q < n && r < r_end) y[(r % Q) * n + p0 + q] = v;
  });
}

// output p of frame r of the window of L samples that starts at absolute sample `start` of a ring (zeros outside the window)
__device__ __forceinline__ float rs_edge_output(const float* __restrict__ ring, long long C, long long start, long long L,
                                                long long r, int p, const float* __restrict__ W, const RsGeom& g) {
  const long long t0 = r * g.o - g.w;
  long long a = (start + t0) % C;
  if (a < 0) a += C;
  const float* wr = W + (size_t)p * g.T;
  float acc = 0.f;
  for (int k = 0; k < g.T; ++k) {
    const long long t = t0 + k;
    const float xv = (t >= 0 && t < L) ? __ldg(ring + a) : 0.f;
    acc = __fmaf_rn(xv, __ldg(wr + k), acc);
    if (++a == C) a = 0;
  }
  return acc;
}

// stream form, second half: window b's frame r is frame r + b * fs of the stream outputs `ys` when all its taps lie inside the
// window (frames r_lo .. r_hi); the frames at the window's edges are recomputed here with the window's zero padding
__global__ void __launch_bounds__(256) resample_assemble_kernel(const float* __restrict__ ring, long long C, long long rpos,
                                                                 long long hop, long long L, const float* __restrict__ ys,
                                                                 long long fs, long long r_lo, long long r_hi,
                                                                 const float* __restrict__ W, RsGeom g, long long out_len,
                                                                 float* __restrict__ out) {
  const int b = blockIdx.y;
  const long long jj = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (jj >= out_len) return;
  const long long r = jj / g.n;
  const int p = (int)(jj - r * g.n);
  float acc;
  if (r >= r_lo && r <= r_hi)
    acc = ys[(r + b * fs) * g.n + p];
  else
    acc = rs_edge_output(ring, C, rpos + b * hop, L, r, p, W, g);
  out[(size_t)b * out_len + jj] = acc;
}

// dg_multi: resampled window rows[i] of the tick batch.  Interior frames r_lo .. r_hi are frames frame0 + r of the slot's
// 16 kHz ring; the edge frames are recomputed from its source ring with the window's zero padding, as the assemble kernel does
__global__ void __launch_bounds__(256) resample_gather_kernel(const float* __restrict__ rings, long long C,
                                                               const float* __restrict__ yrings, long long Y, long long Q,
                                                               const RsRow* __restrict__ rows, long long r_lo, long long r_hi,
                                                               const float* __restrict__ W, RsGeom g, long long L,
                                                               long long out_len, float* __restrict__ wav) {
  const RsRow rw = rows[blockIdx.y];
  const long long jj = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (jj >= out_len) return;
  const long long r = jj / g.n;
  const int p = (int)(jj - r * g.n);
  float v;
  if (r >= r_lo && r <= r_hi)
    v = yrings[(size_t)rw.slot * Y + ((rw.frame0 + r) % Q) * g.n + p];
  else
    v = rs_edge_output(rings + (size_t)rw.slot * C, C, rw.start, L, r, p, W, g);
  wav[(size_t)rw.row * out_len + jj] = v;
}

template <int QF, int QP>
int launch_tile(const RsJob& j, const RsPlan& p, int items, long long max_frames, cudaStream_t st) {
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    DG_CUDA(cudaFuncSetAttribute(resample_tile_kernel<QF, QP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RS_SMEM_MAX));
  const long long gx = (max_frames + p.tile_frames - 1) / p.tile_frames;
  resample_tile_kernel<QF, QP><<<dim3((unsigned)gx, (unsigned)items), RS_THREADS, p.smem, st>>>(j, p.fg);
  DG_LAUNCHED();
  return 0;
}

template <int QF, int QP>
int launch_frames(const float* rings, long long C, const RsFrames* items, int n_items, long long max_count, const float* W,
                  const RsGeom& g, float* yrings, long long Y, long long Q, const RsPlan& p, cudaStream_t st) {
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    DG_CUDA(cudaFuncSetAttribute(resample_frames_kernel<QF, QP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RS_SMEM_MAX));
  const long long gx = (max_count + p.tile_frames - 1) / p.tile_frames;
  resample_frames_kernel<QF, QP><<<dim3((unsigned)gx, (unsigned)n_items), RS_THREADS, p.smem, st>>>(rings, C, items, W, g, yrings,
                                                                                                   Y, Q, p.fg);
  DG_LAUNCHED();
  return 0;
}

}  // namespace

long long resample_out_len(const RsGeom& g, long long L) { return (g.n * L + g.o - 1) / g.o; }

bool resample_geom_ok(const RsGeom& g) { return rs_plan(g).smem <= RS_SMEM_MAX; }

int launch_resample(const RsJob& j, int items, long long max_out, cudaStream_t st) {
  if (items < 1 || max_out < 1) return 0;
  ProfScope _ps("resample", st);
  const RsPlan p = rs_plan(j.g);
  // frames an item's outputs [j_lo, j_lo + j_cnt) may touch: one more than j_cnt / n when j_lo is not frame-aligned
  const long long max_frames = (max_out + j.g.n - 1) / j.g.n + 1;
  return p.qp == 1 ? launch_tile<4, 1>(j, p, items, max_frames, st) : launch_tile<2, 2>(j, p, items, max_frames, st);
}

int launch_resample_stream(const float* ring, long long C, long long rpos, long long hop, long long L, int B, const float* W,
                           const RsGeom& g, float* ys, float* out, cudaStream_t st) {
  const long long out_len = resample_out_len(g, L);
  const long long nfr = (out_len + g.n - 1) / g.n;   // frames per window
  const long long fs = hop / g.o;
  const long long NR = (B - 1) * fs + nfr;
  // every output of the stream once ...
  RsJob j{};
  j.x = ring;
  j.C = C;
  j.base = RsItem{rpos, (B - 1) * hop + L, 0, NR * g.n, 0};
  j.W = W;
  j.g = g;
  j.out = ys;
  int rc;
  if ((rc = launch_resample(j, 1, NR * g.n, st))) return rc;
  // ... then the windows, edge frames recomputed with the window's own zero padding
  ProfScope _ps("resample", st);
  const long long r_lo = (g.w + g.o - 1) / g.o;
  const long long r_hi = L - g.w - g.o >= 0 ? (L - g.w - g.o) / g.o : -1;
  resample_assemble_kernel<<<dim3((unsigned)((out_len + 255) / 256), (unsigned)B), 256, 0, st>>>(ring, C, rpos, hop, L, ys, fs, r_lo,
                                                                                              r_hi, W, g, out_len, out);
  DG_LAUNCHED();
  return 0;
}

int launch_resample_frames(const float* rings, long long C, const RsFrames* items, int n_items, long long max_count,
                           const float* W, const RsGeom& g, float* yrings, long long Y, long long Q, cudaStream_t st) {
  if (n_items < 1 || max_count < 1) return 0;
  if (n_items > 65535) {
    set_error("resample_frames: at most 65535 items per launch");
    return -1;
  }
  ProfScope _ps("resample_frames", st);
  const RsPlan p = rs_plan(g);
  return p.qp == 1 ? launch_frames<4, 1>(rings, C, items, n_items, max_count, W, g, yrings, Y, Q, p, st)
                   : launch_frames<2, 2>(rings, C, items, n_items, max_count, W, g, yrings, Y, Q, p, st);
}

int launch_resample_gather(const float* rings, long long C, const float* yrings, long long Y, long long Q, const RsRow* rows,
                           int n_rows, long long r_lo, long long r_hi, const float* W, const RsGeom& g, long long L,
                           long long out_len, float* wav, cudaStream_t st) {
  if (n_rows < 1) return 0;
  if (n_rows > 65535) {
    set_error("resample_gather: at most 65535 windows per launch");
    return -1;
  }
  ProfScope _ps("resample_gather", st);
  resample_gather_kernel<<<dim3((unsigned)((out_len + 255) / 256), (unsigned)n_rows), 256, 0, st>>>(rings, C, yrings, Y, Q, rows,
                                                                                                 r_lo, r_hi, W, g, L, out_len, wav);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

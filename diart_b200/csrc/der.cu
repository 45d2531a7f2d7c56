// Diarization error rate of hyper-parameter trials on the device (the `metric(reference, hypothesis)` step of the reference's
// Benchmark.evaluate with DiarizationErrorRate, src/diart/inference.py:359-390), DESIGN.md "DER scoring" for the definition:
// collar=0, skip_overlap=False and no uem, or any of them through the scored regions the hypotheses are cropped to.
//
//   der_hyp<false> / der_hyp<true>   one warp per (file, trial, label): walks the sweep's per-chunk turns of that file's
//                                    chunk range in chunk order, with the file's timestamp shift, and merges that label's
//                                    turns into whole-file segments with PredictionAccumulator's collar rule (count pass,
//                                    then write pass at scanned offsets)
//   der_scan                         exclusive prefix sum of the (file, trial, label) counts
//   der_score                        one warp per (file, trial) against that file's reference: k-way merge of the boundary
//                                    lists (one lane per hypothesis label and per reference label), co-occurrence matrix,
//                                    LSAP, the five components; der_score<true, *> first crops each hypothesis label to the
//                                    file's scored pieces (CropList); der_score<*, true> scores the identification error
//                                    rate: no co-occurrence and no LSAP, each reference label's partner is the hypothesis
//                                    label of the same name, from a per-file table
//
// Every float64 operation is explicitly rounded (no FMA contraction): the segment times equal numpy's turn_times /
// assemble_predictions bit for bit, and the components are sums in time order, independent of the launch geometry.
#include "dg_common.cuh"
#include "lsap_warp.cuh"

namespace dg {

constexpr int DER_THREADS = 256;
constexpr int DER_SCORE_THREADS = 128;

// whole-file segments of label g in trial t of file f: turn times as blocks/post.py turn_times, segments with duration <= 1e-6
// dropped, merged in chunk order (= (start, end) order: the chunks' output regions tile the file's timeline) with a running
// maximum of the ends; a segment joins when it starts less than `collar` after that maximum or not after it.  Six CTAs per SM
// (at most 42 registers): without a minimum ptxas holds the kernel to 32 registers and spills in the file loop.
template <bool WRITE>
__global__ void __launch_bounds__(DER_THREADS, 6)
der_hyp_kernel(const int32_t* __restrict__ header /*[T][N][4]*/, const uint32_t* __restrict__ turns, int nf,
               const int* __restrict__ chunk_off /*[nf+1]*/, int T, int N, int M, const double* __restrict__ out_start,
               const double* __restrict__ out_res, const double* __restrict__ shifts /*[nf]*/, double collar,
               int* __restrict__ counts /*[nf*T*M+1]: count pass output, write pass offsets*/, double* __restrict__ segs,
               double* __restrict__ segs_copy, int copy_cap) {
  const int w = (int)(((size_t)blockIdx.x * DER_THREADS + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= nf * T * M) return;   // the whole warp
  const int ft = w / M, g = w - ft * M, f = ft / T, t = ft - f * T;
  const int c_begin = chunk_off[f], c_end = chunk_off[f + 1];
  const double shift = shifts[f];
  const int32_t* hd = header + (size_t)t * N * 4;
  int n = 0, o = WRITE ? counts[w] : 0;
  bool open = false;
  double cs = 0.0, ce = 0.0;
  auto emit = [&]() {
    if (WRITE && lane == 0) {
      segs[(size_t)o * 2] = cs;
      segs[(size_t)o * 2 + 1] = ce;
      if (segs_copy && o < copy_cap) {
        segs_copy[(size_t)o * 2] = cs;
        segs_copy[(size_t)o * 2 + 1] = ce;
      }
    }
    o++;
    n++;
  };
  for (int c0 = c_begin; c0 < c_end; c0 += 32) {
    // lane j finds label g's turns in chunk c0 + j: a chunk's turns are grouped by label in ascending order (post.cu)
    int lo = 0, hi = 0;
    if (c0 + lane < c_end) {
      const int4 h = *reinterpret_cast<const int4*>(hd + (size_t)(c0 + lane) * 4);
      int a = h.x;
      const int e = h.x + h.y;
      while (a < e && (int)(turns[a] >> 20) < g) a++;
      int b = a;
      while (b < e && (int)(turns[b] >> 20) == g) b++;
      lo = a;
      hi = b;
    }
    for (unsigned has = __ballot_sync(FULL, hi > lo); has; has &= has - 1) {
      const int j = __ffs(has) - 1;
      const int a = __shfl_sync(FULL, lo, j), b = __shfl_sync(FULL, hi, j);
      const double s0 = out_start[c0 + j], r0 = out_res[c0 + j];
      for (int i = a; i < b; i++) {
        const uint32_t tw = turns[i];
        const double x = __dadd_rn(s0, __dmul_rn((double)((tw >> 10) & 1023u), r0));
        const double y = __dadd_rn(s0, __dmul_rn((double)(tw & 1023u), r0));
        const double ts = __dadd_rn(__dmul_rn(0.5, __dadd_rn(x, __dadd_rn(x, r0))), shift);   // SlidingWindow[i].middle
        const double te = __dadd_rn(__dmul_rn(0.5, __dadd_rn(y, __dadd_rn(y, r0))), shift);
        if (!(__dsub_rn(te, ts) > 1e-6)) continue;                                            // Segment.__bool__
        if (open && (__dsub_rn(ts, ce) < collar || ts <= ce)) {
          ce = fmax(ce, te);
        } else {
          if (open) emit();
          cs = ts;
          ce = te;
          open = true;
        }
      }
    }
  }
  if (open) emit();
  if (!WRITE && lane == 0) counts[w] = n;
}

// in place: counts [n] -> exclusive offsets [n + 1]; one CTA of 1024 threads, each scanning a contiguous slice
__global__ void __launch_bounds__(1024) der_scan_kernel(int* __restrict__ counts, int n) {
  __shared__ int part[1024];
  const int per = (n + 1023) / 1024, a = min(n, (int)threadIdx.x * per), b = min(n, a + per);
  int s = 0;
  for (int i = a; i < b; i++) s += counts[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const int v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  int run = part[threadIdx.x] - s;
  for (int i = a; i < b; i++) {
    const int c = counts[i];
    counts[i] = run;
    run += c;
  }
  if (threadIdx.x == 1023) counts[n] = part[1023];
}

// one label's sorted, disjoint segments, read one at a time; `b` is the current boundary
struct SegList {
  const double* p;
  int i, n;
  double s, e;
  __device__ void load() {
    if (i < n) {
      s = p[(size_t)i * 2];
      e = p[(size_t)i * 2 + 1];
    }
  }
  __device__ void advance(double b) {   // drop the segments that end at or before b
    while (i < n && e <= b) {
      i++;
      load();
    }
  }
  __device__ bool active(double b) const { return i < n && s <= b; }
  __device__ double next(double b) const { return i < n ? (s > b ? s : e) : INFINITY; }
};

// One hypothesis label's segments cropped to the file's scored pieces (DESIGN.md "DER scoring", step 4), read one piece at a
// time with SegList's interface: segment i is cut against each scored piece k it intersects (Segment.intersects with
// pyannote.core's 1e-6 s precision, in float64 as oracle/detection.py has it), and a falsy intersection is dropped.  The
// label's segments are sorted and apart, so its pieces are too.  j: the first scored piece that does not end at or before
// segment i's start; k: the next candidate for segment i.
struct CropList {
  const double* p;
  int i, n;
  const double* u;
  int j, m, k;
  double hs, he, s, e;
  __device__ void start_segment() {
    hs = p[(size_t)i * 2];
    he = p[(size_t)i * 2 + 1];
    while (j < m && u[(size_t)j * 2 + 1] <= hs) j++;
    k = j;
  }
  __device__ void seek() {   // from candidate (i, k) on, to the next truthy piece (i = n: none)
    while (i < n) {
      if (k < m && u[(size_t)k * 2] < he) {
        const double bs = u[(size_t)k * 2], be = u[(size_t)k * 2 + 1];
        k++;
        const bool hit = (hs < bs && bs < __dsub_rn(he, 1e-6)) || (hs > bs && hs < __dsub_rn(be, 1e-6)) || hs == bs;
        const double cs = fmax(hs, bs), ce = fmin(he, be);
        if (hit && __dsub_rn(ce, cs) > 1e-6) {
          s = cs;
          e = ce;
          return;
        }
      } else if (++i < n) {
        start_segment();
      }
    }
  }
  __device__ void load() {
    if (i < n) start_segment();
    seek();
  }
  __device__ void advance(double b) {
    while (i < n && e <= b) seek();
  }
  __device__ bool active(double b) const { return i < n && s <= b; }
  __device__ double next(double b) const { return i < n ? (s > b ? s : e) : INFINITY; }
};

// Walks the elementary intervals [b, bn) of the union of all boundaries in time order and calls body(d, hyp active, ref active)
// for each one with Segment(b, bn) truthy.  Lane l holds hypothesis label l (`hl`: a SegList, or a CropList) and reference
// label l.
template <typename HypList, typename Body>
__device__ __forceinline__ void der_walk_list(HypList& hl, SegList& rl, Body body) {
  hl.load();
  rl.load();
  double b = warp_min_d(fmin(hl.next(-INFINITY), rl.next(-INFINITY)));
  while (b < INFINITY) {
    hl.advance(b);
    rl.advance(b);
    const bool ah = hl.active(b), ar = rl.active(b);
    const double bn = warp_min_d(fmin(hl.next(b), rl.next(b)));
    if (bn == INFINITY) break;
    const double d = __dsub_rn(bn, b);
    if (d > 1e-6) body(d, ah, ar);
    b = bn;
  }
}

// der_walk_list over hypothesis segments [h0, h1) of hp, cropped to the scored pieces [u0, u1) of up when CROP
template <bool CROP, typename Body>
__device__ __forceinline__ void der_walk(const double* hp, int h0, int h1, const double* up, int u0, int u1,
                                         const double* rp, int r0, int r1, Body body) {
  if constexpr (CROP) {
    CropList hl{hp, h0, h1, up, u0, u1, 0, 0.0, 0.0, 0.0, 0.0};
    SegList rl{rp, r0, r1, 0.0, 0.0};
    der_walk_list(hl, rl, body);
  } else {
    SegList hl{hp, h0, h1, 0.0, 0.0}, rl{rp, r0, r1, 0.0, 0.0};
    der_walk_list(hl, rl, body);
  }
}

// comp [nf][T][5] = {false alarm, missed detection, confusion, correct, total}; warp (f, t) scores trial t of file f against
// file f's reference: R[f] labels at offsets roff [f][DER_ROFF] into rseg.  CROP: every hypothesis label is first cropped to
// file f's scored pieces [uoff[f], uoff[f + 1]) of useg (CropList); the reference comes cropped from the host.  NAMED (the
// identification error rate, DESIGN.md "Identification error"): reference label r of file f is matched to hypothesis label
// named [f][r] (-1: none) instead of the LSAP's partner; pass 2 is the same.
template <bool CROP, bool NAMED>
__global__ void __launch_bounds__(DER_SCORE_THREADS)
der_score_kernel(const int* __restrict__ hoff /*[nf*T*M+1]*/, const double* __restrict__ hseg, int nf, int T, int M,
                 const int* __restrict__ roff_all /*[nf][DER_ROFF]*/, const int* __restrict__ R_all /*[nf]*/,
                 const double* __restrict__ rseg, double* __restrict__ comp, const int* __restrict__ uoff /*[nf+1]*/,
                 const double* __restrict__ useg, const int* __restrict__ named /*[nf][32]*/) {
  __shared__ double tr[DER_SCORE_THREADS / 32][32][33];
  const int ft = (int)(((size_t)blockIdx.x * DER_SCORE_THREADS + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (ft >= nf * T) return;
  const int f = ft / T, R = R_all[f];
  const int* roff = roff_all + (size_t)f * DER_ROFF;
  const int h0 = lane < M ? hoff[ft * M + lane] : 0, h1 = lane < M ? hoff[ft * M + lane + 1] : 0;
  const int r0 = lane < R ? roff[lane] : 0, r1 = lane < R ? roff[lane + 1] : 0;
  const int u0 = CROP ? uoff[f] : 0, u1 = CROP ? uoff[f + 1] : 0;
  int partner = -1;   // lane r: the hypothesis label mapped to reference label r
  if constexpr (NAMED) {
    if (lane < R) partner = named[(size_t)f * 32 + lane];
  } else {
  // pass 1: co-occurrence C[r][h], lane h owns column h, each entry summed in time order
  double C[32];
#pragma unroll
  for (int q = 0; q < 32; q++) C[q] = 0.0;
  der_walk<CROP>(hseg, h0, h1, useg, u0, u1, rseg, r0, r1, [&](double d, bool ah, bool ar) {
    const unsigned rmask = __ballot_sync(FULL, ar);
#pragma unroll
    for (int q = 0; q < 32; q++)
      if (ah && ((rmask >> q) & 1u)) C[q] = __dadd_rn(C[q], d);
  });
  // the one-to-one mapping of maximal total co-occurrence: LSAP on -C, rows = the smaller side (scipy transposes a tall matrix)
  if (R > 0) {
    double(&s)[32][33] = tr[threadIdx.x >> 5];
#pragma unroll
    for (int q = 0; q < 32; q++) s[q][lane] = C[q];
    __syncwarp();
    const bool rows_ref = R <= M;
#pragma unroll
    for (int q = 0; q < 32; q++) C[q] = -(rows_ref ? s[q][lane] : s[lane][q]);
    __syncwarp();
    const int c4r = lsap_warp(C, rows_ref ? R : M, rows_ref ? M : R, lane);
    if (rows_ref) {
      partner = lane < R ? c4r : -1;
    } else {
      for (int h = 0; h < M; h++) {
        const int r = __shfl_sync(FULL, c4r, h);
        if (lane == r) partner = h;
      }
    }
  }
  }
  // pass 2: the components, in time order
  double fa = 0.0, miss = 0.0, conf = 0.0, corr = 0.0, tot = 0.0;
  der_walk<CROP>(hseg, h0, h1, useg, u0, u1, rseg, r0, r1, [&](double d, bool ah, bool ar) {
    const unsigned hmask = __ballot_sync(FULL, ah);
    const int nr = __popc(__ballot_sync(FULL, ar)), nh = __popc(hmask);
    const int c = __popc(__ballot_sync(FULL, ar && partner >= 0 && ((hmask >> partner) & 1u)));
    tot = __dadd_rn(tot, __dmul_rn(d, (double)nr));
    miss = __dadd_rn(miss, __dmul_rn(d, (double)max(0, nr - nh)));
    fa = __dadd_rn(fa, __dmul_rn(d, (double)max(0, nh - nr)));
    corr = __dadd_rn(corr, __dmul_rn(d, (double)c));
    conf = __dadd_rn(conf, __dmul_rn(d, (double)(min(nr, nh) - c)));
  });
  if (lane == 0) {
    double* o = comp + (size_t)ft * 5;
    o[0] = fa;
    o[1] = miss;
    o[2] = conf;
    o[3] = corr;
    o[4] = tot;
  }
}

int launch_der_hyp_count(const int32_t* header, const uint32_t* turns, int nf, const int* chunk_off, int T, int N, int M,
                         const double* out_start, const double* out_res, const double* shifts, double collar, int* offsets,
                         cudaStream_t st) {
  ProfScope _ps("der_hyp_count", st);
  const long long warps = (long long)nf * T * M;
  const unsigned blocks = (unsigned)((warps * 32 + DER_THREADS - 1) / DER_THREADS);
  der_hyp_kernel<false><<<blocks, DER_THREADS, 0, st>>>(header, turns, nf, chunk_off, T, N, M, out_start, out_res, shifts,
                                                         collar, offsets, nullptr, nullptr, 0);
  DG_LAUNCHED();
  der_scan_kernel<<<1, 1024, 0, st>>>(offsets, (int)warps);
  DG_LAUNCHED();
  return 0;
}

int launch_der_hyp_write(const int32_t* header, const uint32_t* turns, int nf, const int* chunk_off, int T, int N, int M,
                         const double* out_start, const double* out_res, const double* shifts, double collar, int* offsets,
                         double* segs, double* segs_copy, int copy_cap, cudaStream_t st) {
  ProfScope _ps("der_hyp_write", st);
  const long long warps = (long long)nf * T * M;
  const unsigned blocks = (unsigned)((warps * 32 + DER_THREADS - 1) / DER_THREADS);
  der_hyp_kernel<true><<<blocks, DER_THREADS, 0, st>>>(header, turns, nf, chunk_off, T, N, M, out_start, out_res, shifts,
                                                        collar, offsets, segs, segs_copy, copy_cap);
  DG_LAUNCHED();
  return 0;
}

int launch_der_score(const int* hoff, const double* hseg, int nf, int T, int M, const int* roff, const int* R,
                     const double* rseg, double* comp, cudaStream_t st, const int* uoff, const double* useg, const int* named) {
  ProfScope _ps("der_score", st);
  const unsigned blocks = (unsigned)(((long long)nf * T * 32 + DER_SCORE_THREADS - 1) / DER_SCORE_THREADS);
  if (uoff && named)
    der_score_kernel<true, true><<<blocks, DER_SCORE_THREADS, 0, st>>>(hoff, hseg, nf, T, M, roff, R, rseg, comp, uoff, useg,
                                                                      named);
  else if (uoff)
    der_score_kernel<true, false><<<blocks, DER_SCORE_THREADS, 0, st>>>(hoff, hseg, nf, T, M, roff, R, rseg, comp, uoff, useg,
                                                                       nullptr);
  else if (named)
    der_score_kernel<false, true><<<blocks, DER_SCORE_THREADS, 0, st>>>(hoff, hseg, nf, T, M, roff, R, rseg, comp, nullptr,
                                                                       nullptr, named);
  else
    der_score_kernel<false, false><<<blocks, DER_SCORE_THREADS, 0, st>>>(hoff, hseg, nf, T, M, roff, R, rseg, comp, nullptr,
                                                                        nullptr, nullptr);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

// Gallery naming: the nearest enrolled speaker of every unnamed global speaker, in float64 (DESIGN.md "Gallery naming").
//
//   gallery_norms    one warp per entry: |e| in float64, once, when the gallery is uploaded.
//   gallery_queries  one CTA: the multi-stream queries of a tick (active, unnamed speakers of the slots with windows and a
//                    gallery), compacted in the host's group order (group, then slot, then speaker), and each group's query
//                    offset and count.
//   gallery_nearest  one CTA per work item (group, query tile, split) of gallery_plan: the group's gallery, entries and norms
//                    from its descriptor; an item whose tile lies beyond the group's query count exits at once.
//                    CTA tile = 64 entries x 128 queries, 8 warps of 32 x 32; both operands staged through shared memory with
//                    cp.async (two stages of 16 columns), dot products on the float64 tensor cores (mma.sync m16n8k4 f64,
//                    sm_90).  The epilogue turns each dot product into the cosine distance, skips claimed entries and keeps per
//                    query the lexicographic minimum (distance, entry) over the CTA's split of the gallery.
//   gallery_claim    one warp per claim group: the minimum over its group's splits, the group's threshold, and the conflicts
//                    within the claim group.
//
// Every dot product is accumulated over k in one fixed order (k-chunks in order, the k-steps of a chunk in order), with no
// atomics, so two identical gallery rows give bit-identical distances and the lowest index wins their tie.  Nothing in that
// order depends on the group, the query tile or the split a query runs in, so a query's distance to an entry is the same
// whether its gallery is searched alone (dg_gallery_query) or as one group among many in a tick.
#include <math.h>

#include <algorithm>

#include "dg_common.cuh"

namespace dg {

namespace {

constexpr int LDS = GAL_KC + 4;     // shared row stride in doubles: the 8 rows x 4 columns of a fragment load hit distinct banks
constexpr int NT = 256;             // 8 warps: 2 along the entries x 4 along the queries
constexpr int SMEM_A = 2 * GAL_TILE_E * LDS, SMEM_B = 2 * GAL_TILE_Q * LDS;   // doubles
// operands, query norms, claim masks, claims, then the CTA's group descriptor and work item (in the dynamic allocation:
// with a static __shared__ block beside it the kernel ran 18 % slower on the H100)
constexpr size_t SMEM_BYTES = (size_t)(SMEM_A + SMEM_B + GAL_TILE_Q) * 8 + (size_t)GAL_TILE_Q * 8 + (size_t)GAL_TILE_Q * 32 * 4 +
                              sizeof(GalGroup) + 8 * 4;

__device__ __forceinline__ bool lex_less(double d1, int e1, double d2, int e2) {
  return d1 < d2 || (d1 == d2 && (unsigned)e1 < (unsigned)e2);
}

__device__ __forceinline__ double cosine_distance(double dot, double nu, double nv) {
  double c = dot / (nu * nv);
  if (fabs(c) > 1.0) c = copysign(1.0, c);
  return 1.0 - c;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// D = A (16 x 4, row) B (4 x 8, col) + D, float64 (PTX ISA: mma.m16n8k4 with .f64, sm_90).  Fragments, g = lane / 4,
// t = lane % 4: a = {A[g][t], A[g + 8][t]}, b = B[t][g], d = {D[g][2t], D[g][2t + 1], D[g + 8][2t], D[g + 8][2t + 1]}.
__device__ __forceinline__ void mma_f64(double (&d)[4], double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a0), "d"(a1), "d"(b));
}

__global__ void __launch_bounds__(256) gallery_norms_kernel(const double* __restrict__ E, int G, int Dp, double* __restrict__ En) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= G) return;
  const double* e = E + (size_t)warp * Dp;
  double s = 0.0;
  for (int d = lane; d < Dp; d += 32) s = fma(e[d], e[d], s);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) En[warp] = sqrt(s);
}

// one CTA of 1024 threads; thread i owns the segments [i per, (i + 1) per)
__global__ void __launch_bounds__(1024) gallery_queries_kernel(const int2* __restrict__ segs, int n_seg,
                                                               const GalGroup* __restrict__ groups, int n_groups,
                                                               const int* __restrict__ active, const uint32_t* __restrict__ named,
                                                               int M, int2* __restrict__ qd, int* __restrict__ seg_off,
                                                               int2* __restrict__ gq, int* __restrict__ names) {
  __shared__ int scan[1024];
  const int tid = threadIdx.x, per = (n_seg + 1023) / 1024, a0 = min(n_seg, tid * per), a1 = min(n_seg, a0 + per);
  auto pending = [&](int a) {
    const int slot = segs[a].x;
    unsigned m = 0;
    for (int g = 0; g < M; g++) m |= (active[slot * 32 + g] != 0 ? 1u : 0u) << g;
    return m & ~named[slot];
  };
  int n = 0;
  for (int a = a0; a < a1; a++) n += __popc(pending(a));
  scan[tid] = n;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {   // inclusive Hillis-Steele scan
    const int v = tid >= o ? scan[tid - o] : 0;
    __syncthreads();
    scan[tid] += v;
    __syncthreads();
  }
  int q = scan[tid] - n;
  for (int a = a0; a < a1; a++) {
    const int slot = segs[a].x;
    seg_off[a] = q;
    for (unsigned m = pending(a); m; m &= m - 1) qd[q++] = make_int2(slot * M + __ffs(m) - 1, slot);
  }
  if (tid == 1023) {
    seg_off[n_seg] = scan[1023];
    names[0] = 0;
  }
  __syncthreads();   // seg_off is complete (block scope)
  for (int r = tid; r < n_groups; r += 1024) {
    const int b = seg_off[groups[r].seg0];
    gq[r] = make_int2(b, seg_off[groups[r].seg1] - b);
  }
}

struct NearestArgs {
  const GalGroup* groups;
  const GalWork* work;
  const int2* gq;
  const double* X;
  const int2* qd;
  const int32_t* claimed;
  double* part_d;
  int* part_e;
  int Dp, D, Qmax;
};

// two CTAs per SM: at most 128 registers (the shared memory of two fits as well)
__global__ void __launch_bounds__(NT, 2) gallery_nearest_kernel(const NearestArgs p) {
  extern __shared__ __align__(16) double smem[];
  double* sA = smem;                                   // [2][64][LDS]
  double* sB = sA + SMEM_A;                            // [2][128][LDS]
  double* qn = sB + SMEM_B;                            // [128] query norms
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(qn + GAL_TILE_Q);   // [128] claimed rows of the tile
  int* claims = reinterpret_cast<int*>(mask + GAL_TILE_Q);                            // [128][32]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp & 1, wn = warp >> 1;             // warp tile: entries wm*32 .., queries wn*32 ..
  // the work item: query tile w.tile of group w.group (queries [gq.x, gq.x + gq.y)) against split w.split of its gallery.
  // The item and its group's descriptor live in shared memory and are read where they are used, so that they hold no
  // registers across the tile loop
  GalGroup& gr = *reinterpret_cast<GalGroup*>(claims + GAL_TILE_Q * 32);
  int* cta = reinterpret_cast<int*>(&gr + 1);   // the tile's first query, the group's query end, the split, its tile range
  {
    const GalWork w = p.work[blockIdx.x];
    const int2 gq = p.gq[w.group];
    if (w.tile * GAL_TILE_Q >= gq.y) return;
    if (tid == 0) {
      gr = p.groups[w.group];
      cta[0] = gq.x + w.tile * GAL_TILE_Q;
      cta[1] = gq.x + gq.y;
      cta[2] = w.split;
      cta[3] = w.split * gr.per_split;
      cta[4] = min(gr.tiles, cta[3] + gr.per_split);
    }
    __syncthreads();
  }
  const int nq = cta[1], q0 = cta[0];
  // the tile's queries: norms (one warp per 16 queries, a fixed order) and their groups' claims
  for (int c = warp; c < GAL_TILE_Q; c += NT / 32) {
    const int q = q0 + c;
    double s = 0.0;
    int grp = -1;
    if (q < nq) {
      const int2 d = p.qd[q];
      grp = d.y;
      const double* x = p.X + (size_t)d.x * p.D;
      for (int k = lane; k < p.D; k += 32) s = fma(x[k], x[k], s);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) qn[c] = q < nq ? sqrt(s) : 0.0;
    claims[c * 32 + lane] = (q < nq && p.claimed) ? p.claimed[(size_t)grp * 32 + lane] : -1;
  }
  // operand rows this thread copies: A rows (tid / 8) and + 32, B rows (tid / 8) + 32 j, column pair 2 (tid % 8)
  const int cr = tid >> 3, cc = (tid & 7) * 2;
  // row offsets into X in 32 bits (fewer registers than pointers): callers keep rows * D <= INT_MAX (dg_gallery_query
  // splits larger calls; a dg_multi's centroid table is at most 65 535 slots x 25 600 = max_speakers x D doubles)
  int xrow[4];
  bool xok[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int q = q0 + cr + 32 * j;
    xok[j] = q < nq;
    xrow[j] = xok[j] ? p.qd[q].x * p.D : 0;
  }
  double best_d[8];
  int best_e[8];
#pragma unroll
  for (int i = 0; i < 8; i++) best_d[i] = INFINITY, best_e[i] = -1;
  const int nk = p.Dp / GAL_KC;
  __syncthreads();
  for (int tile = cta[3]; tile < cta[4]; tile++) {
    const int e0 = tile * GAL_TILE_E;
    if (tid < GAL_TILE_Q) {
      unsigned long long m = 0;
      for (int j = 0; j < 32; j++) {
        const int e = claims[tid * 32 + j] - e0;
        if (e >= 0 && e < GAL_TILE_E) m |= 1ull << e;
      }
      mask[tid] = m;
    }
    auto load = [&](int kc, int stage) {
      const int k = kc * GAL_KC + cc;
      double* a = sA + stage * GAL_TILE_E * LDS;
      double* b = sB + stage * GAL_TILE_Q * LDS;
#pragma unroll
      for (int j = 0; j < 2; j++)
        cp_async16(a + (cr + 32 * j) * LDS + cc, gr.E + (size_t)(e0 + cr + 32 * j) * p.Dp + k, true);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const bool ok = xok[j] && k < p.D;
        cp_async16(b + (cr + 32 * j) * LDS + cc, p.X + (ok ? (size_t)(xrow[j] + k) : 0), ok);
      }
      cp_async_commit();
    };
    double acc[2][4][4];
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
#pragma unroll
        for (int i = 0; i < 4; i++) acc[mi][ni][i] = 0.0;
    load(0, 0);
    for (int kc = 0; kc < nk; kc++) {
      if (kc + 1 < nk) {
        load(kc + 1, (kc + 1) & 1);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      const double* a = sA + (kc & 1) * GAL_TILE_E * LDS + (wm * 32 + g) * LDS + t;
      const double* b = sB + (kc & 1) * GAL_TILE_Q * LDS + (wn * 32 + g) * LDS + t;
#pragma unroll
      for (int ks = 0; ks < GAL_KC; ks += 4) {
        double af[2][2], bf[4];
#pragma unroll
        for (int mi = 0; mi < 2; mi++) af[mi][0] = a[(mi * 16) * LDS + ks], af[mi][1] = a[(mi * 16 + 8) * LDS + ks];
#pragma unroll
        for (int ni = 0; ni < 4; ni++) bf[ni] = b[(ni * 8) * LDS + ks];
#pragma unroll
        for (int mi = 0; mi < 2; mi++)
#pragma unroll
          for (int ni = 0; ni < 4; ni++) mma_f64(acc[mi][ni], af[mi][0], af[mi][1], bf[ni]);
      }
      __syncthreads();
    }
    // epilogue: entry row wm*32 + mi*16 + g (+8 for i >= 2), query column wn*32 + ni*8 + 2t + (i & 1)
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r = wm * 32 + mi * 16 + g + 8 * h, e = e0 + r;
        if (e >= gr.G) continue;
        const double en = gr.En[e];
#pragma unroll
        for (int ni = 0; ni < 4; ni++)
#pragma unroll
          for (int j = 0; j < 2; j++) {
            const int c = wn * 32 + ni * 8 + 2 * t + j;
            if ((mask[c] >> r) & 1ull) continue;
            const double d = cosine_distance(acc[mi][ni][2 * h + j], qn[c], en);
            if (lex_less(d, e, best_d[ni * 2 + j], best_e[ni * 2 + j])) best_d[ni * 2 + j] = d, best_e[ni * 2 + j] = e;
          }
      }
    __syncthreads();   // mask is rewritten by the next tile
  }
  // reduce over the 8 row groups of the warp (lanes with the same t), then over the two warps along the entries
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      const double d = __shfl_xor_sync(0xffffffffu, best_d[i], o);
      const int e = __shfl_xor_sync(0xffffffffu, best_e[i], o);
      if (lex_less(d, e, best_d[i], best_e[i])) best_d[i] = d, best_e[i] = e;
    }
  double* red_d = sA;                                             // [2][128]
  int* red_e = reinterpret_cast<int*>(sA + 2 * GAL_TILE_Q);       // [2][128]
  if (g == 0)
#pragma unroll
    for (int ni = 0; ni < 4; ni++)
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int c = wn * 32 + ni * 8 + 2 * t + j;
        red_d[wm * GAL_TILE_Q + c] = best_d[ni * 2 + j];
        red_e[wm * GAL_TILE_Q + c] = best_e[ni * 2 + j];
      }
  __syncthreads();
  if (tid < GAL_TILE_Q && cta[0] + tid < cta[1]) {
    double d = red_d[tid];
    int e = red_e[tid];
    if (lex_less(red_d[GAL_TILE_Q + tid], red_e[GAL_TILE_Q + tid], d, e)) d = red_d[GAL_TILE_Q + tid], e = red_e[GAL_TILE_Q + tid];
    const size_t o = (size_t)cta[2] * p.Qmax + cta[0] + tid;
    p.part_d[o] = d;
    p.part_e[o] = e;
  }
}

__global__ void __launch_bounds__(128) gallery_claim_kernel(const double* __restrict__ part_d, const int* __restrict__ part_e,
                                                            int Qmax, const int2* __restrict__ qd, const int* __restrict__ seg_off,
                                                            const int2* __restrict__ segs, int n_seg,
                                                            const GalGroup* __restrict__ groups, int32_t* claimed,
                                                            int32_t* entry_out, double* dist_out, uint32_t* named, int M,
                                                            int* names, int32_t* list, int32_t* prefix) {
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= n_seg) return;
  const int off = seg_off[s], cnt = seg_off[s + 1] - off;
  if (cnt <= 0) return;
  const GalGroup& grp = groups[segs[s].y];
  const int splits = grp.splits;
  const double threshold = grp.threshold;
  const int q = off + lane;
  double d = INFINITY;
  int e = -1;
  if (lane < cnt)
    for (int k = 0; k < splits; k++) {
      const double dk = part_d[(size_t)k * Qmax + q];
      const int ek = part_e[(size_t)k * Qmax + q];
      if (ek >= 0 && lex_less(dk, ek, d, e)) d = dk, e = ek;
    }
  const int cand = (e >= 0 && d < threshold) ? e : -1;
  bool win = cand >= 0;
  for (int k = 0; k < 32; k++) {      // another candidate for the same entry that is closer, or as close and earlier
    const int ck = __shfl_sync(0xffffffffu, cand, k);
    const double dk = __shfl_sync(0xffffffffu, d, k);
    if (k != lane && ck == cand && (dk < d || (dk == d && k < lane))) win = false;
  }
  if (lane < cnt && entry_out) {
    entry_out[q] = win ? cand : -1;
    dist_out[q] = d;
  }
  if (!named) return;
  const int2 qq = lane < cnt ? qd[q] : make_int2(0, 0);
  const int r = qq.y, gg = qq.x - qq.y * M;
  const unsigned ballot = __ballot_sync(0xffffffffu, win);
  if (!ballot) return;
  int base = 0;
  if (lane == 0) base = atomicAdd(names, __popc(ballot));
  base = __shfl_sync(0xffffffffu, base, 0);
  const unsigned bits = __reduce_or_sync(0xffffffffu, win ? 1u << gg : 0u);
  if (win) {
    claimed[(size_t)r * 32 + gg] = cand;
    const int i = base + __popc(ballot & ((1u << lane) - 1));
    const int32_t rec[3] = {r, gg, cand};
    for (int j = 0; j < 3; j++) list[3 * i + j] = rec[j];
    if (i < GAL_NAME_PREFIX)
      for (int j = 0; j < 3; j++) prefix[3 * i + j] = rec[j];
  }
  if (lane == __ffs(ballot) - 1) named[r] |= bits;
}

}  // namespace

int launch_gallery_norms(const double* E, int G, int Dp, double* En, cudaStream_t st) {
  ProfScope _ps("gallery_norms", st);
  gallery_norms_kernel<<<(unsigned)(((long long)G * 32 + 255) / 256), 256, 0, st>>>(E, G, Dp, En);
  DG_LAUNCHED();
  return 0;
}

int gallery_plan(std::vector<GalGroup>& groups, std::vector<GalWork>& work) {
  work.clear();
  int qtiles = 0, splits = 0;
  std::vector<int> busy;   // the groups with queries: every split loop below visits only them, so the plan is O(groups + work)
  for (int r = 0; r < (int)groups.size(); r++) {
    qtiles += (groups[r].q_ub + GAL_TILE_Q - 1) / GAL_TILE_Q;
    if (groups[r].q_ub > 0) busy.push_back(r);
  }
  const int s = qtiles ? std::min((2 * 132 + qtiles - 1) / qtiles, 64) : 1;   // about two CTAs per SM
  for (GalGroup& g : groups) {
    g.tiles = (g.G + GAL_TILE_E - 1) / GAL_TILE_E;
    // as many tiles in every split, and no split empty
    const int per = (g.tiles + std::min(s, g.tiles) - 1) / std::min(s, g.tiles);
    g.splits = (g.tiles + per - 1) / per;
    g.per_split = (g.tiles + g.splits - 1) / g.splits;
    if (g.q_ub > 0) splits = std::max(splits, g.splits);
  }
  work.reserve((size_t)qtiles * splits);
  for (int k = 0; k < splits; k++)
    for (int r : busy)
      if (k < groups[r].splits)
        for (int t = 0; t < (groups[r].q_ub + GAL_TILE_Q - 1) / GAL_TILE_Q; t++) work.push_back(GalWork{r, t, k});
  return splits;
}

int launch_gallery_nearest(const GalGroup* groups, const GalWork* work, int n_work, const int2* gq, int Dp, const double* X,
                           int D, const int2* qd, int Qmax, const int32_t* claimed, double* part_d, int* part_e,
                           cudaStream_t st) {
  ProfScope _ps("gallery_nearest", st);
  if (n_work <= 0) return 0;
  static bool attr[64] = {};
  if (first_use_on_device(attr))
    DG_CUDA(cudaFuncSetAttribute(gallery_nearest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  const NearestArgs p{groups, work, gq, X, qd, claimed, part_d, part_e, Dp, D, Qmax};
  gallery_nearest_kernel<<<(unsigned)n_work, NT, SMEM_BYTES, st>>>(p);
  DG_LAUNCHED();
  return 0;
}

int launch_gallery_queries(const int2* segs, int n, const GalGroup* groups, int n_groups, const int* active,
                           const uint32_t* named, int M, int2* qd, int* seg_off, int2* gq, int* names, cudaStream_t st) {
  ProfScope _ps("gallery_queries", st);
  gallery_queries_kernel<<<1, 1024, 0, st>>>(segs, n, groups, n_groups, active, named, M, qd, seg_off, gq, names);
  DG_LAUNCHED();
  return 0;
}

int launch_gallery_claim(const double* part_d, const int* part_e, int Qmax, const int2* qd, const int* seg_off,
                         const int2* segs, int n_seg, const GalGroup* groups, int32_t* claimed, int32_t* entry_out,
                         double* dist_out, uint32_t* named, int M, int* names, int32_t* list, int32_t* prefix, cudaStream_t st) {
  ProfScope _ps("gallery_claim", st);
  if (n_seg <= 0) return 0;
  gallery_claim_kernel<<<(unsigned)(((long long)n_seg * 32 + 127) / 128), 128, 0, st>>>(
      part_d, part_e, Qmax, qd, seg_off, segs, n_seg, groups, claimed, entry_out, dist_out, named, M, names, list, prefix);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

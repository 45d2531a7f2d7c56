// OnlineSpeakerClustering on the device (float64 + int, bit-exact decision logic).
//
// Restates reference src/diart/blocks/clustering.py:119-218 (identify / __call__) and the SpeakerMap
// operations it reaches in src/diart/mapping.py:179-360: every mutation (unmap_speakers,
// unmap_threshold, set_source_speaker) yields a NEW cost matrix whose Hungarian assignment is
// re-solved lazily; here a "map" is a (K x M) float64 matrix held one column per lane of warp 0, and
// `solve()` is scipy.optimize.linear_sum_assignment's algorithm (Crouse 2016 shortest augmenting
// path, the published algorithm behind scipy's rectangular LSAP) executed column-parallel with
// scipy's tie-breaking order reproduced exactly (oracle/lsap_ref.py is the same restatement in
// Python, fuzzed against scipy).
//
// Two kernels per batch:
//   cluster_prep  (parallel over chunks)  per-speaker max / mean of the segmentation, NaN flags and
//                                         float64 norms of the embeddings.
//   cluster_seq   (one CTA per state)     walks the B chunks in order: float64 cosine distances to
//                                         the active centroids (8 warps), the assignment logic
//                                         (warp 0), then centroid update + SpeakerMap.apply scatter
//                                         (all threads).
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "dg_common.cuh"
#include "lsap_warp.cuh"

namespace dg {

constexpr int CK = 8;          // max local speakers
constexpr int CM = 32;         // max global speakers (one per lane)
constexpr double INVALID = 1e10;

size_t cluster_prep_floats(int B, int K) { return (size_t)B * K * 3; }     // max, mean, nan flag
size_t cluster_prep_doubles(int B, int K) { return (size_t)B * K; }        // ||e||

// numpy semantics: np.max / np.mean over axis 0 of a float32 (F,K) array.  The mean is a float32
// running sum in frame order followed by one float32 division (clustering.py:137-142).  Chunk i; shared by cluster_prep_kernel
// and cluster_prep_sets_kernel.
__device__ __forceinline__ void cluster_prep_chunk(const float* __restrict__ seg, const float* __restrict__ emb, int i, int F,
                                                   int K, int D, float* __restrict__ prep, double* __restrict__ prep_d) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* s = seg + (size_t)i * F * K;
  if (threadIdx.x < K) {
    float mx = -INFINITY, sum = 0.f;
    for (int f = 0; f < F; f++) {
      const float v = s[f * K + threadIdx.x];
      mx = (isnan(v) || isnan(mx)) ? NAN : fmaxf(mx, v);   // np.max propagates NaN (fmaxf alone would drop it again)
      sum = __fadd_rn(sum, v);
    }
    prep[((size_t)i * K + threadIdx.x) * 3 + 0] = mx;
    prep[((size_t)i * K + threadIdx.x) * 3 + 1] = __fdiv_rn(sum, (float)F);
  }
  for (int k = warp; k < K; k += 4) {
    const float* e = emb + ((size_t)i * K + k) * D;
    double ss = 0.0;
    int nan = 0;
    for (int d = lane; d < D; d += 32) {
      const float v = e[d];
      nan |= isnan(v);
      ss = fma((double)v, (double)v, ss);
    }
    for (int o = 16; o > 0; o >>= 1) {
      ss += __shfl_xor_sync(FULL, ss, o);
      nan |= __shfl_xor_sync(FULL, nan, o);
    }
    if (lane == 0) {
      prep[((size_t)i * K + k) * 3 + 2] = nan ? 1.f : 0.f;
      prep_d[(size_t)i * K + k] = sqrt(ss);
    }
  }
}

__global__ void __launch_bounds__(128) cluster_prep_kernel(const float* __restrict__ seg, const float* __restrict__ emb,
                                                           int F, int K, int D, float* __restrict__ prep,
                                                           double* __restrict__ prep_d) {
  cluster_prep_chunk(seg, emb, blockIdx.x, F, K, D, prep, prep_d);
}

// one CTA per (chunk, set) over the embeddings of G sets [G][B][K][D]: set g's rows at prep + g B K 3 and prep_d + g B K (the
// score statistics are the same in every set)
__global__ void __launch_bounds__(128) cluster_prep_sets_kernel(const float* __restrict__ seg, const float* __restrict__ emb,
                                                                int F, int K, int D, float* __restrict__ prep,
                                                                double* __restrict__ prep_d) {
  const size_t g = blockIdx.y, B = gridDim.x;
  cluster_prep_chunk(seg, emb + g * B * K * D, blockIdx.x, F, K, D, prep + g * B * K * 3, prep_d + g * B * K);
}

__device__ __forceinline__ void put(double (&c)[CK], int i, double v) {
#pragma unroll
  for (int q = 0; q < CK; q++) c[q] = (i == q) ? v : c[q];
}

struct SeqShared {
  double dist[CK][CM];
  int map[CK];
  int upd_k[CK], upd_g[CK], n_upd;   // centers[g] += emb[k]
  int new_k[CK], new_g[CK], n_new;   // centers[g]  = emb[k]
  int active[CM];
  int initialized;
  int error;
};

// mapped rows of a cost matrix held one column per lane: bit k set iff min_j C[k][j] != 1e10
__device__ __forceinline__ unsigned mapped_rows(const double (&c)[CK], int K, int M, int lane) {
  unsigned m = 0;
#pragma unroll
  for (int k = 0; k < CK; k++) {
    if (k < K) {
      const bool any = __any_sync(FULL, lane < M && c[k] != INVALID);
      if (any) m |= 1u << k;
    }
  }
  return m;
}

__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem));
}

constexpr int SEQ_THREADS = 512;        // one stream's state: the pipeline
constexpr int SWEEP_THREADS = 256;      // many independent states (hyper-parameter sweep): 2 CTAs per SM by registers

// One CTA per clustering state.  STATES = false compiles the single-state form of the pipeline (grid of one, the thresholds
// of `p`, no per-state indexing).  STATES = true: CTA i runs the state states[i] = {file f, trial t} over the chunks
// [chunk_off[f], chunk_off[f + 1]) of the B concatenated ones, with {tau, rho, delta} = trials [t] (float64); state
// s = f T + t owns centroid table s ([M][D] at centers + s M D), active flags s ([32]) and the `initialized` / error pair s,
// and writes the map rows of its chunks in trial t's block ([B][K] at map_out + t B K).  Outputs are addressed by (f, t),
// so the launch order (the order of `states`) changes no result.  OWN_ROWS (STATES only; many live streams, each at its own
// thresholds, dg_multi): t is only the row of `trials`, state s = f, and every state's maps go to block 0.  The arithmetic
// does not depend on THREADS: each centroid's distances are one warp's, the updates are element-wise.  SETS (STATES only; sweeps
// over OSP sets): a trial row is {tau, rho, delta, set} and the state reads the embeddings and prep rows of that set, emb
// [G][B][K][D], prep [G][B][K][3], prep_d [G][B][K] (64-bit offsets: G B K D exceeds 2^31 on large datasets).
template <int THREADS, bool STATES, bool OWN_ROWS = false, bool SETS = false>
__global__ void __launch_bounds__(THREADS)
cluster_seq_kernel(ClusterParams p, const double* __restrict__ trials, const int2* __restrict__ states,
                   const int* __restrict__ chunk_off, int T, const float* __restrict__ seg,
                   const float* __restrict__ emb, int B, int F, int K, double* __restrict__ centers,
                   int* __restrict__ g_active, int* __restrict__ g_init, const float* __restrict__ prep,
                   const double* __restrict__ prep_d, int32_t* __restrict__ map_out, float* __restrict__ permuted,
                   unsigned* __restrict__ dbg) {
  constexpr int SEQ_THREADS = THREADS;
  __shared__ SeqShared sh;
  __shared__ float prs[2][CK * 3];      // per-chunk max / mean / nan flag, double buffered
  __shared__ double ens[2][CK];         // per-chunk embedding norms
  extern __shared__ __align__(16) unsigned char dyn[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int M = p.M, D = p.D;
  constexpr int NW = SEQ_THREADS / 32;
  float tau_f = p.tau_f, rho_f = p.rho_f;
  double delta = p.delta;
  int first = 0;                                // chunk ci of this state is chunk first + ci of seg / emb / prep
  if constexpr (STATES) {
    const int2 fs = states[blockIdx.x];
    const int trial = fs.y, c0 = chunk_off[fs.x];
    constexpr int PS = SETS ? 4 : 3;                     // doubles per trial row
    if constexpr (SETS) {
      const size_t set = (size_t)trials[trial * PS + 3], n = (size_t)B * K;   // B: all chunks of the launch here
      emb += set * n * p.D;
      prep += set * n * 3;
      prep_d += set * n;
    }
    const size_t s = OWN_ROWS ? (size_t)fs.x : (size_t)fs.x * T + trial;
    centers += s * M * D;
    g_active += s * CM;
    g_init += s * 2;
    map_out += ((size_t)(OWN_ROWS ? 0 : trial) * B + c0) * K;
    B = chunk_off[fs.x + 1] - c0;              // from here on: this file's chunks, the first at c0
    first = c0;
    // numpy compares the float32 scores with a Python float in float32 (as dg_cluster_create)
    tau_f = (float)trials[trial * PS + 0];
    rho_f = (float)trials[trial * PS + 1];
    delta = trials[trial * PS + 2];
  }
  double* cs = reinterpret_cast<double*>(dyn);                 // centroids [M][D], resident for the whole batch
  double* ed = cs + (size_t)M * D;                             // the current chunk's embeddings as float64 [K][D] (converted once
                                                               // per chunk by all threads instead of once per centroid warp)
  float* es = reinterpret_cast<float*>(ed + (size_t)K * D);    // embeddings [2][K][D], double buffered (cp.async landing zone)
  auto prefetch = [&](int ci, int buf) {
    const size_t cg = (size_t)(first + ci);
    const float* e = emb + cg * K * D;
    for (int i = tid; i < K * D; i += SEQ_THREADS) cp_async4(es + (size_t)buf * K * D + i, e + i);
    if (tid < K * 3) cp_async4(&prs[buf][tid], prep + cg * K * 3 + tid);
    if (tid < K * 2) cp_async4(reinterpret_cast<float*>(&ens[buf][0]) + tid,
                               reinterpret_cast<const float*>(prep_d + cg * K) + tid);
    asm volatile("cp.async.commit_group;");
  };
  prefetch(0, 0);
  for (int i = tid; i < M * D; i += SEQ_THREADS) cs[i] = centers[i];
  if (tid < CM) sh.active[tid] = tid < M ? g_active[tid] : 0;
  if (tid == 0) {
    sh.initialized = *g_init;
    sh.error = 0;
  }
  asm volatile("cp.async.wait_group 0;");
  __syncthreads();
  for (int i = tid; i < K * D; i += SEQ_THREADS) ed[i] = (double)es[i];
  __syncthreads();

  for (int ci = 0; ci < B; ci++) {
    const int cur = ci & 1;
    const float* ecur = es + (size_t)cur * K * D;
    const float* pr = prs[cur];
    const bool init = sh.initialized != 0;
    if (dbg && tid == 0) dbg[ci * 4 + 0] = (unsigned)clock();
    if (ci + 1 < B) prefetch(ci + 1, cur ^ 1);
    // ---------------- phase A: float64 cosine distances (scipy cdist 'cosine':
    //                  1 - u.v / (|u| |v|), clipped to [-1, 1] before the subtraction).
    //                  One warp per active centroid: its norm and its K dot products in one pass.
    if (init && p.metric == 0) {
      for (int g = warp; g < M; g += NW) {
        if (!sh.active[g]) continue;
        const double* c = cs + (size_t)g * D;
        double acc[CK + 1];
#pragma unroll
        for (int k = 0; k <= CK; k++) acc[k] = 0.0;
#pragma unroll 4
        for (int d = lane; d < D; d += 32) {
          const double cv = c[d];
          acc[CK] = fma(cv, cv, acc[CK]);
#pragma unroll
          for (int k = 0; k < CK; k++)
            if (k < K) acc[k] = fma(ed[k * D + d], cv, acc[k]);
        }
#pragma unroll
        for (int k = 0; k <= CK; k++)
          if (k < K || k == CK)
            for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(FULL, acc[k], o);
        // lane k finishes local speaker k: ONE float64 square root and ONE division per warp, executed by all lanes at once (a
        // branch per k would run the three divisions one after the other: the float64 division is a long dependent chain)
        double dot = acc[0];
#pragma unroll
        for (int k = 1; k < CK; k++) dot = (lane == k) ? acc[k] : dot;
        const double en = ens[cur][lane < K ? lane : 0];
        double cosv = dot / (en * sqrt(acc[CK]));
        if (fabs(cosv) > 1.0) cosv = copysign(1.0, cosv);
        if (lane < K) sh.dist[lane][g] = 1.0 - cosv;
      }
    } else if (init) {
      // the other scipy.spatial.distance.cdist metrics the reference accepts through `metric` (mapping.py:175), in float64:
      // 1 euclidean, 2 sqeuclidean, 3 cityblock, 4 chebyshev
      for (int g = warp; g < M; g += NW) {
        if (!sh.active[g]) continue;
        const double* c = cs + (size_t)g * D;
        double acc[CK];
#pragma unroll
        for (int k = 0; k < CK; k++) acc[k] = 0.0;
        for (int d = lane; d < D; d += 32) {
          const double cv = c[d];
#pragma unroll
          for (int k = 0; k < CK; k++)
            if (k < K) {
              const double df = ed[k * D + d] - cv;
              if (p.metric <= 2) acc[k] = fma(df, df, acc[k]);
              else if (p.metric == 3) acc[k] += fabs(df);
              else acc[k] = fmax(acc[k], fabs(df));
            }
        }
#pragma unroll
        for (int k = 0; k < CK; k++)
          if (k < K)
            for (int o = 16; o > 0; o >>= 1) {
              const double other = __shfl_xor_sync(FULL, acc[k], o);
              acc[k] = p.metric == 4 ? fmax(acc[k], other) : acc[k] + other;
            }
#pragma unroll
        for (int k = 0; k < CK; k++)
          if (k < K && lane == k) sh.dist[k][g] = p.metric == 1 ? sqrt(acc[k]) : acc[k];
      }
    }
    __syncthreads();
    // ---------------- phase B: assignment logic, warp 0, one global speaker per lane
    if (warp == 0) {
      if (dbg && lane == 0) dbg[ci * 4 + 1] = (unsigned)clock();
      unsigned active_spk = 0, long_spk = 0;
      for (int k = 0; k < K; k++) {
        // np.max(seg) >= tau, np.mean(seg) >= rho: float32 array vs Python float -> float32 compare
        if (pr[k * 3 + 0] >= tau_f && pr[k * 3 + 2] == 0.f) active_spk |= 1u << k;   // clustering.py:137-145
        if (pr[k * 3 + 1] >= rho_f) long_spk |= 1u << k;
      }
      int n_upd = 0, n_new = 0;
      if (!init) {                                                                      // clustering.py:149-158
        int next = 0;
        for (int k = 0; k < K; k++) {
          int g = -1;
          if ((active_spk >> k) & 1u) {
            g = next++;
            if (lane == 0) {
              sh.new_k[n_new] = k;
              sh.new_g[n_new] = g;
            }
            n_new++;
            if (lane == g) sh.active[g] = 1;
          }
          if (lane == 0) sh.map[k] = g;
        }
        if (lane == 0) sh.initialized = 1;
      } else {
        const bool act_c = lane < M && sh.active[lane];
        const int n_active = __popc(__ballot_sync(FULL, act_c));
        double dmap[CK], valid[CK];
#pragma unroll
        for (int k = 0; k < CK; k++) {                                                  // clustering.py:161-166
          const bool live = k < K && ((active_spk >> k) & 1u) && act_c;
          dmap[k] = live ? sh.dist[k][lane] : INVALID;
          valid[k] = dmap[k];
        }
        // unmap_threshold (mapping.py:260-273)
        int c4r = lsap_warp(dmap, K, M, lane);
        unsigned mapped = mapped_rows(dmap, K, M, lane);
        bool dirty = false;
        for (int k = 0; k < K; k++) {
          if (!((mapped >> k) & 1u)) continue;
          const int c = __shfl_sync(FULL, c4r, k);
          const double cost = __shfl_sync(FULL, sel(dmap, k), c);
          if (cost >= delta) {
            put(valid, k, INVALID);
            dirty = true;
          }
        }
        unsigned vmapped = mapped_rows(valid, K, M, lane);
        const unsigned missed = active_spk & ~vmapped;                                  // clustering.py:171-173
        const int n_free = M - n_active;   // blocked_centers is always empty (clustering.py:46)
        unsigned new_mask = 0;
        for (int k = 0; k < K; k++) {                                                   // clustering.py:176-194
          if (!((missed >> k) & 1u)) continue;
          if (n_new < n_free && ((long_spk >> k) & 1u)) {
            n_new++;
            new_mask |= 1u << k;
          } else {
            if (dirty) {
              c4r = lsap_warp(valid, K, M, lane);
              dirty = false;
            }
            vmapped = mapped_rows(valid, K, M, lane);
            unsigned tk = 0;
            for (int q = 0; q < K; q++) {
              const int cq = __shfl_sync(FULL, c4r, q);
              if ((vmapped >> q) & 1u) tk |= 1u << cq;
            }
            // closest active centre that is not already a target
            const bool ok = act_c && !((tk >> lane) & 1u);
            const double dk = ok ? sel(dmap, k) : INFINITY;
            const double best = warp_min_d(dk);
            const unsigned who = __ballot_sync(FULL, ok && dk == best);
            if (who) {
              const int g = __ffs(who) - 1;
              if (lane == g) put(valid, k, 0.0);                                        // mapping.py:245-251
              dirty = true;
            }
          }
        }
        if (dirty) {
          c4r = lsap_warp(valid, K, M, lane);
          dirty = false;
        }
        vmapped = mapped_rows(valid, K, M, lane);
        for (int k = 0; k < K; k++) {                                                   // clustering.py:197-202
          if (!((vmapped >> k) & 1u) || ((missed >> k) & 1u) || !((long_spk >> k) & 1u)) continue;
          const int g = __shfl_sync(FULL, c4r, k);
          if (!sh.active[g]) {
            if (lane == 0) sh.error = 1;   // reference: AssertionError("Cannot update unknown centers")
            continue;
          }
          if (lane == 0) {
            sh.upd_k[n_upd] = k;
            sh.upd_g[n_upd] = g;
          }
          n_upd++;
        }
        // new centres at the lowest free index (clustering.py:205-208, 68-71)
        int q = 0;
        for (int k = 0; k < K; k++) {
          if (!((new_mask >> k) & 1u)) continue;
          const unsigned freeb = __ballot_sync(FULL, lane < M && !sh.active[lane]);
          const int g = __ffs(freeb) - 1;
          if (lane == g) {
            sh.active[g] = 1;
            put(valid, k, 0.0);
          }
          if (lane == 0) {
            sh.new_k[q] = k;
            sh.new_g[q] = g;
          }
          q++;
          dirty = true;
          __syncwarp();
        }
        if (dirty) c4r = lsap_warp(valid, K, M, lane);
        vmapped = mapped_rows(valid, K, M, lane);
        if (lane < K) sh.map[lane] = ((vmapped >> lane) & 1u) ? c4r : -1;
      }
      if (lane == 0) {
        sh.n_upd = n_upd;
        sh.n_new = n_new;
        if (dbg) dbg[ci * 4 + 2] = (unsigned)clock();
      }
    }
    __syncthreads();
    // ---------------- phase C: centroid update / creation, outputs
    for (int q = 0; q < sh.n_upd; q++) {
      double* c = cs + (size_t)sh.upd_g[q] * D;
      const float* e = ecur + (size_t)sh.upd_k[q] * D;
      for (int d = tid; d < D; d += SEQ_THREADS) c[d] += (double)e[d];
    }
    for (int q = 0; q < sh.n_new; q++) {
      double* c = cs + (size_t)sh.new_g[q] * D;
      const float* e = ecur + (size_t)sh.new_k[q] * D;
      for (int d = tid; d < D; d += SEQ_THREADS) c[d] = (double)e[d];
    }
    if (tid < K) map_out[(size_t)ci * K + tid] = sh.map[tid];
    if (permuted) {                                                                     // mapping.py:341-360
      float* o = permuted + (size_t)ci * F * M;
      const float* s = seg + (size_t)(first + ci) * F * K;
      for (int idx = tid; idx < F * M; idx += SEQ_THREADS) o[idx] = 0.f;
      __syncthreads();
      for (int k = 0; k < K; k++) {
        const int g = sh.map[k];
        if (g < 0) continue;
        for (int f = tid; f < F; f += SEQ_THREADS) o[(size_t)f * M + g] = s[f * K + k];
      }
    }
    asm volatile("cp.async.wait_group 0;");
    __syncthreads();
    if (ci + 1 < B) {            // the next chunk's embeddings have landed: float64 copies for its distance phase
      const float* enext = es + (size_t)(cur ^ 1) * K * D;
      for (int i = tid; i < K * D; i += SEQ_THREADS) ed[i] = (double)enext[i];
      __syncthreads();
    }
    if (dbg && tid == 0) dbg[ci * 4 + 3] = (unsigned)clock();
  }
  for (int i = tid; i < M * D; i += SEQ_THREADS) centers[i] = cs[i];
  if (tid < M) g_active[tid] = sh.active[tid];
  if (tid == 0) {
    *g_init = sh.initialized;
    if (sh.error) g_init[1] = 1;
  }
}

// bytes of dynamic shared memory one state needs: centroids, the current chunk's embeddings as float64, the double-buffered
// float32 landing zone
static size_t cluster_seq_dyn(int M, int D, int K) {
  return (size_t)M * D * sizeof(double) + (size_t)K * D * sizeof(double) + (size_t)2 * K * D * sizeof(float);
}

static int check_cluster_shape(const char* who, const ClusterParams& p, int K) {
  if (K > CK || p.M > CM || K > p.M) {
    set_error(std::string(who) + ": need local speakers <= 8, max_speakers <= 32 and local <= max");
    return -1;
  }
  if (cluster_seq_dyn(p.M, p.D, K) > 200 * 1024) {
    set_error(std::string(who) + ": max_speakers * dim too large for the resident centroid table (limit 200 KB)");
    return -1;
  }
  return 0;
}

template <int THREADS, bool STATES, bool OWN_ROWS = false, bool SETS = false>
static int cluster_seq_allow_dyn() {   // per device: the opt-in above 48 KB is a property of (function, device)
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done))
    DG_CUDA(cudaFuncSetAttribute(cluster_seq_kernel<THREADS, STATES, OWN_ROWS, SETS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 200 * 1024));
  return 0;
}

int launch_cluster_step(const ClusterParams& p, const float* seg, const float* emb, int B, int F, int K,
                        double* centers, int* active, int* initialized, float* prep, double* prep_d, int32_t* map,
                        float* permuted, cudaStream_t st) {
  ProfScope _ps("cluster_step", st);
  if (check_cluster_shape("cluster_step", p, K)) return -1;
  if (B <= 0) return 0;
  cluster_prep_kernel<<<B, 128, 0, st>>>(seg, emb, F, K, p.D, prep, prep_d);
  DG_LAUNCHED();
  const size_t dyn = cluster_seq_dyn(p.M, p.D, K);
  if (int rc = cluster_seq_allow_dyn<SEQ_THREADS, false>()) return rc;
  static const bool timing = getenv("DG_CLUSTER_TIMING") && getenv("DG_CLUSTER_TIMING")[0] == '1';
  if (timing) {   // diagnostic: SM-clock stamps per chunk (distances | assignment logic | update + hand-over), synchronises
    unsigned* dbg = nullptr;
    DG_CUDA(cudaMalloc(&dbg, (size_t)B * 4 * sizeof(unsigned)));
    cluster_seq_kernel<SEQ_THREADS, false><<<1, SEQ_THREADS, dyn, st>>>(p, nullptr, nullptr, nullptr, 1, seg, emb, B, F, K, centers,
                                                                active, initialized, prep, prep_d, map, permuted, dbg);
    DG_CUDA(cudaStreamSynchronize(st));
    std::vector<unsigned> hb((size_t)B * 4);
    DG_CUDA(cudaMemcpy(hb.data(), dbg, hb.size() * 4, cudaMemcpyDeviceToHost));
    cudaFree(dbg);
    double a = 0, b = 0, c = 0;
    for (int i = 0; i < B; i++) {
      a += (double)(int)(hb[i * 4 + 1] - hb[i * 4 + 0]);
      b += (double)(int)(hb[i * 4 + 2] - hb[i * 4 + 1]);
      c += (double)(int)(hb[i * 4 + 3] - hb[i * 4 + 2]);
    }
    static int shown = 0;
    if (shown++ < 8)
      fprintf(stderr, "cluster_seq timing (B=%d, cycles per chunk): distances %.0f | assignment logic %.0f | update + hand-over %.0f | total %.0f\n",
              B, a / B, b / B, c / B, (a + b + c) / B);
    DG_LAUNCHED();
    return 0;
  }
  cluster_seq_kernel<SEQ_THREADS, false><<<1, SEQ_THREADS, dyn, st>>>(p, nullptr, nullptr, nullptr, 1, seg, emb, B, F, K, centers,
                                                              active, initialized, prep, prep_d, map, permuted, nullptr);
  DG_LAUNCHED();
  return 0;
}

// S independent (file, trial) states over the B concatenated chunks of the files, each from its trial's {tau, rho, delta}
// (trials_dev [T][3] float64): one prep pass over all B chunks, then one CTA per state in the order of states_dev.  States
// beyond the resident CTAs run in later waves of the same launch.
int launch_cluster_sweep(const ClusterParams& p, const double* trials_dev, int T, const int2* states_dev, int S,
                         const int* chunk_off_dev, const float* seg, const float* emb, int B, int F, int K, double* centers,
                         int* active, int* initialized, float* prep, double* prep_d, int32_t* maps, cudaStream_t st,
                         bool own_rows) {
  ProfScope _ps("cluster_sweep", st);
  if (check_cluster_shape("cluster_sweep", p, K)) return -1;
  if (B <= 0 || S <= 0) return 0;
  cluster_prep_kernel<<<B, 128, 0, st>>>(seg, emb, F, K, p.D, prep, prep_d);
  DG_LAUNCHED();
  const size_t dyn = cluster_seq_dyn(p.M, p.D, K);
  if (own_rows) {
    if (int rc = cluster_seq_allow_dyn<SWEEP_THREADS, true, true>()) return rc;
    cluster_seq_kernel<SWEEP_THREADS, true, true><<<S, SWEEP_THREADS, dyn, st>>>(
        p, trials_dev, states_dev, chunk_off_dev, T, seg, emb, B, F, K, centers, active, initialized, prep, prep_d, maps,
        nullptr, nullptr);
  } else {
    if (int rc = cluster_seq_allow_dyn<SWEEP_THREADS, true>()) return rc;
    cluster_seq_kernel<SWEEP_THREADS, true><<<S, SWEEP_THREADS, dyn, st>>>(
        p, trials_dev, states_dev, chunk_off_dev, T, seg, emb, B, F, K, centers, active, initialized, prep, prep_d, maps,
        nullptr, nullptr);
  }
  DG_LAUNCHED();
  return 0;
}

int launch_cluster_sweep_sets(const ClusterParams& p, const double* trials_dev, int T, const int2* states_dev, int S,
                              const int* chunk_off_dev, const float* seg, const float* emb, int G, int B, int F, int K,
                              double* centers, int* active, int* initialized, float* prep, double* prep_d, int32_t* maps,
                              cudaStream_t st) {
  ProfScope _ps("cluster_sweep", st);
  if (check_cluster_shape("cluster_sweep", p, K)) return -1;
  if (B <= 0 || S <= 0) return 0;
  cluster_prep_sets_kernel<<<dim3(B, G), 128, 0, st>>>(seg, emb, F, K, p.D, prep, prep_d);
  DG_LAUNCHED();
  const size_t dyn = cluster_seq_dyn(p.M, p.D, K);
  if (int rc = cluster_seq_allow_dyn<SWEEP_THREADS, true, false, true>()) return rc;
  cluster_seq_kernel<SWEEP_THREADS, true, false, true><<<S, SWEEP_THREADS, dyn, st>>>(
      p, trials_dev, states_dev, chunk_off_dev, T, seg, emb, B, F, K, centers, active, initialized, prep, prep_d, maps,
      nullptr, nullptr);
  DG_LAUNCHED();
  return 0;
}

// One CTA per sweep state s = f T + t: copies file f's known centroids into rows 0 .. n_f - 1 of centroid table s and marks
// them active; the state counts as initialised when n_f > 0, so cluster_seq takes the distance path from its first chunk (the
// reference's identify with `centers` already set).  Tables of states whose file has no centroids stay as zeroed.
__global__ void __launch_bounds__(256) sweep_seed_kernel(const int* __restrict__ seed_off, const double* __restrict__ seeds,
                                                         int T, int M, int D, double* __restrict__ centers,
                                                         int* __restrict__ active, int* __restrict__ initialized) {
  const size_t s = blockIdx.x;
  const int f = (int)(s / T), a = seed_off[f], n = seed_off[f + 1] - a;
  if (n == 0) return;
  const double* src = seeds + (size_t)a * D;
  double* dst = centers + s * M * D;
  for (int i = threadIdx.x; i < n * D; i += blockDim.x) dst[i] = src[i];
  if ((int)threadIdx.x < n) active[s * CM + threadIdx.x] = 1;
  if (threadIdx.x == 0) initialized[s * 2] = 1;
}

int launch_sweep_seed(const int* seed_off, const double* seeds, int nf, int T, int M, int D, double* centers, int* active,
                      int* initialized, cudaStream_t st) {
  ProfScope _ps("sweep_seed", st);
  if (nf <= 0 || T <= 0) return 0;
  sweep_seed_kernel<<<(unsigned)((long long)nf * T), 256, 0, st>>>(seed_off, seeds, T, M, D, centers, active, initialized);
  DG_LAUNCHED();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// Shared-identity mode (extension beyond the reference, SURVEY.md 8(e) / BASELINE config 5): G ranks diarize
// independent streams against ONE table of global speakers.  After every pipeline step each rank exports a
// fixed-size record of what it changed since the last merge, the records are all-gathered (one NCCL collective of
// M*(D+1)+2 doubles per rank) and every rank applies all of them in rank order with the same rule, so all ranks
// hold bit-identical tables again.
//   record = [M][D] payload, [M] kind, 2 reserved;  kind 0: untouched / inactive, 1: payload = centroid - base
//   (centre existed at the last merge), 2: payload = a centre this rank CREATED during the step.
// Merge: base += deltas (rank order); then every created centre, in (rank, index) order: a rank already judged its
// creation new w.r.t. every centre it could see, so only centres created by EARLIER ranks in this merge are
// candidates for being the same speaker (cosine distance < delta_new -> summed into it); otherwise it takes the
// lowest free index; with a full table it joins the closest centre.  Creations of one rank stay distinct.
// `relabel` tells the calling rank where each of its own created centres ended up (identity for the rest).
__global__ void __launch_bounds__(128) cluster_export_kernel(const double* __restrict__ centers, const int* __restrict__ active,
                                                             const double* __restrict__ base, const int* __restrict__ base_active,
                                                             int M, int D, double* __restrict__ record) {
  const int g = blockIdx.x;
  const int kind = !active[g] ? 0 : (base_active[g] ? 1 : 2);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const double c = centers[(size_t)g * D + d];
    record[(size_t)g * D + d] = kind == 1 ? c - base[(size_t)g * D + d] : (kind == 2 ? c : 0.0);
  }
  if (threadIdx.x == 0) {
    record[(size_t)M * D + g] = (double)kind;
    if (g == 0) record[(size_t)M * D + M] = record[(size_t)M * D + M + 1] = 0.0;
  }
}

__global__ void __launch_bounds__(256) cluster_merge_kernel(const double* __restrict__ records, int world, int rank, int M, int D,
                                                            int rec_len, double delta_new, double* __restrict__ centers,
                                                            int* __restrict__ active, double* __restrict__ base,
                                                            int* __restrict__ base_active, int* __restrict__ initialized,
                                                            int32_t* __restrict__ relabel) {
  __shared__ int s_active[CM], s_fresh[CM], s_used[CM];
  __shared__ double s_dist[CM];
  __shared__ int s_target;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < CM) {
    s_active[tid] = tid < M ? base_active[tid] : 0;
    s_fresh[tid] = 0;
  }
  if (tid < M) relabel[tid] = tid;
  for (int i = tid; i < M * D; i += blockDim.x) centers[i] = base[i];
  __syncthreads();
  // 1. updates of centres that existed at the last merge, rank order
  for (int r = 0; r < world; r++) {
    const double* rec = records + (size_t)r * rec_len;
    for (int g = 0; g < M; g++) {
      if (rec[(size_t)M * D + g] != 1.0) continue;
      for (int d = tid; d < D; d += blockDim.x) centers[(size_t)g * D + d] += rec[(size_t)g * D + d];
    }
  }
  __syncthreads();
  // 2. centres created during the step, (rank, index) order
  for (int r = 0; r < world; r++) {
    const double* rec = records + (size_t)r * rec_len;
    __syncthreads();
    if (tid < CM) s_used[tid] = 0;
    __syncthreads();
    for (int g = 0; g < M; g++) {
      if (rec[(size_t)M * D + g] != 2.0) continue;
      const double* c = rec + (size_t)g * D;
      for (int a = warp; a < M; a += 8) {     // cosine distance to every active centre (warp per centre)
        double dot = 0.0, na = 0.0, nc = 0.0;
        if (s_active[a])
          for (int d = lane; d < D; d += 32) {
            const double x = centers[(size_t)a * D + d], y = c[d];
            dot = fma(x, y, dot);
            na = fma(x, x, na);
            nc = fma(y, y, nc);
          }
        for (int o = 16; o > 0; o >>= 1) {
          dot += __shfl_xor_sync(FULL, dot, o);
          na += __shfl_xor_sync(FULL, na, o);
          nc += __shfl_xor_sync(FULL, nc, o);
        }
        if (lane == 0) {
          double dist = INFINITY;
          if (s_active[a]) {
            double cosv = dot / (sqrt(nc) * sqrt(na));
            if (fabs(cosv) > 1.0) cosv = copysign(1.0, cosv);
            dist = 1.0 - cosv;
          }
          s_dist[a] = dist;
        }
      }
      __syncthreads();
      if (tid == 0) {
        int best = -1, free_idx = -1;
        double bd = INFINITY;
        for (int a = 0; a < M; a++)
          if (!s_active[a] && free_idx < 0) free_idx = a;
        for (int a = 0; a < M; a++) {
          const bool cand = s_active[a] && !s_used[a] && (free_idx < 0 || s_fresh[a]);
          if (cand && s_dist[a] < bd) {
            bd = s_dist[a];
            best = a;
          }
        }
        int target = -1;
        if (best >= 0 && (bd < delta_new || free_idx < 0)) target = best;
        else if (free_idx >= 0) target = free_idx;
        s_target = target;
      }
      __syncthreads();
      const int target = s_target;
      if (target < 0) continue;            // full table and every centre already taken by this rank's creations
      if (s_active[target]) {
        for (int d = tid; d < D; d += blockDim.x) centers[(size_t)target * D + d] += c[d];
      } else {
        for (int d = tid; d < D; d += blockDim.x) centers[(size_t)target * D + d] = c[d];
      }
      __syncthreads();
      if (tid == 0) {
        if (!s_active[target]) s_fresh[target] = 1;
        s_active[target] = 1;
        s_used[target] = 1;
        if (r == rank) relabel[g] = target;
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < M * D; i += blockDim.x) base[i] = centers[i];
  if (tid < M) {
    active[tid] = s_active[tid];
    base_active[tid] = s_active[tid];
  }
  if (tid == 0) {
    int any = 0;
    for (int a = 0; a < M; a++) any |= s_active[a];
    if (any) *initialized = 1;
  }
}

__global__ void relabel_maps_kernel(int32_t* __restrict__ maps, int n, const int32_t* __restrict__ relabel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && maps[i] >= 0) maps[i] = relabel[maps[i]];
}

int launch_cluster_export(const double* centers, const int* active, const double* base, const int* base_active, int M,
                          int D, double* record, cudaStream_t st) {
  ProfScope _ps("cluster_export", st);
  cluster_export_kernel<<<M, 128, 0, st>>>(centers, active, base, base_active, M, D, record);
  DG_LAUNCHED();
  return 0;
}

int launch_cluster_merge(const double* records, int world, int rank, const ClusterParams& p, int rec_len, double* centers,
                         int* active, double* base, int* base_active, int* initialized, int32_t* relabel,
                         cudaStream_t st) {
  ProfScope _ps("cluster_merge", st);
  cluster_merge_kernel<<<1, 256, 0, st>>>(records, world, rank, p.M, p.D, rec_len, p.delta, centers, active, base,
                                          base_active, initialized, relabel);
  DG_LAUNCHED();
  return 0;
}

int launch_relabel_maps(int32_t* maps, int n, const int32_t* relabel, cudaStream_t st) {
  ProfScope _ps("relabel_maps", st);
  relabel_maps_kernel<<<(n + 255) / 256, 256, 0, st>>>(maps, n, relabel);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

// Small fused kernels either side of the two networks:
//   seg_final   PyanNet classifier Linear(128,K) + sigmoid                      (SURVEY.md App. A.3)
//   osp         OverlappedSpeechPenalty      reference src/diart/functional.py:6-13,
//                                            src/diart/blocks/embedding.py:98-107
//   stats_pool  pyannote StatsPool with (resized) weights, K poolings per trunk pass   (App. A.5)
//   l2norm      EmbeddingNormalization       reference src/diart/functional.py:16-27
//   row flags / gather for the (N,1,S)-repeated compatibility entry
//                                            reference src/diart/blocks/embedding.py:57-59
#include "dg_common.cuh"

namespace dg {

// ------------------------------------------------------------------------------------- seg_final
template <int KMAX>
__global__ void __launch_bounds__(256) seg_final_kernel(const float* __restrict__ y, const float* __restrict__ wc,
                                                        const float* __restrict__ bc, int T, int stride, int K,
                                                        float* __restrict__ seg) {
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 w[KMAX];
  float bias[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; k++) {
    w[k] = k < K ? *reinterpret_cast<const float4*>(wc + k * 128 + lane * 4) : make_float4(0, 0, 0, 0);
    bias[k] = k < K ? bc[k] : 0.f;
  }
  for (int t = warp; t < T; t += 8) {
    const float4 v = *reinterpret_cast<const float4*>(y + ((size_t)b * stride + t) * 128 + lane * 4);
#pragma unroll
    for (int k = 0; k < KMAX; k++) {
      if (k >= K) break;
      float d = v.x * w[k].x;
      d = fmaf(v.y, w[k].y, d);
      d = fmaf(v.z, w[k].z, d);
      d = fmaf(v.w, w[k].w, d);
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (lane == 0) seg[((size_t)b * T + t) * K + k] = 1.f / (1.f + expf(-(d + bias[k])));
    }
  }
}

int launch_seg_final(const float* y, const float* wc, const float* bc, int B, int T, int stride, int K, float* seg,
                     cudaStream_t st) {
  ProfScope _ps("seg_final", st);
  if (K > 8) {
    set_error("seg_final: at most 8 local speakers");
    return -1;
  }
  if (K <= 4) seg_final_kernel<4><<<B, 256, 0, st>>>(y, wc, bc, T, stride, K, seg);
  else seg_final_kernel<8><<<B, 256, 0, st>>>(y, wc, bc, T, stride, K, seg);
  DG_LAUNCHED();
  return 0;
}

// powerset models (pyannote/segmentation-3.0): Linear(128, C) -> log_softmax over C classes (= subsets of the local
// speakers of size <= max_per_frame) -> Powerset.to_multilabel = one_hot(argmax) @ mapping, i.e. hard {0,1} scores
// (reference PowersetAdapter, src/diart/models.py:29-39).  argmax of log_softmax = argmax of the logits (first maximum,
// like torch.argmax); `masks[c]` = speaker bit set of class c.
__global__ void __launch_bounds__(256) seg_powerset_kernel(const float* __restrict__ y, const float* __restrict__ wc,
                                                           const float* __restrict__ bc, int T, int stride, int C,
                                                           int num_speakers, const unsigned* __restrict__ masks,
                                                           float* __restrict__ seg) {
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 w[8];
  float bias[8];
#pragma unroll
  for (int k = 0; k < 8; k++) {
    w[k] = k < C ? *reinterpret_cast<const float4*>(wc + k * 128 + lane * 4) : make_float4(0, 0, 0, 0);
    bias[k] = k < C ? bc[k] : 0.f;
  }
  for (int t = warp; t < T; t += 8) {
    const float4 v = *reinterpret_cast<const float4*>(y + ((size_t)b * stride + t) * 128 + lane * 4);
    int best = 0;
    float best_v = -INFINITY;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      if (k >= C) break;
      float d = v.x * w[k].x;
      d = fmaf(v.y, w[k].y, d);
      d = fmaf(v.z, w[k].z, d);
      d = fmaf(v.w, w[k].w, d);
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      d += bias[k];
      if (d > best_v) {     // strict: the first maximum wins
        best_v = d;
        best = k;
      }
    }
    if (lane < num_speakers) seg[((size_t)b * T + t) * num_speakers + lane] = (masks[best] >> lane) & 1u ? 1.f : 0.f;
  }
}

int launch_seg_powerset(const float* y, const float* wc, const float* bc, int B, int T, int stride, int C, int num_speakers,
                        const unsigned* masks_dev, float* seg, cudaStream_t st) {
  ProfScope _ps("seg_final", st);
  if (C > 8 || num_speakers > 8) {
    set_error("seg_powerset: at most 8 classes / speakers");
    return -1;
  }
  seg_powerset_kernel<<<B, 256, 0, st>>>(y, wc, bc, T, stride, C, num_speakers, masks_dev, seg);
  DG_LAUNCHED();
  return 0;
}

// ------------------------------------------------------------------------------------------- osp
__device__ __forceinline__ float pow_like_torch(float x, float g) {
  if (g == 3.f) return x * x * x;
  if (g == 2.f) return x * x;
  if (g == 1.f) return x;
  return powf(x, g);
}

// Item b of an OSP launch: weights for all frames staged in shared memory so the optional min-max normalisation over frames
// (embedding.py:102-106) needs no second launch.  Shared by osp_kernel and osp_sets_kernel.
__device__ __forceinline__ void osp_item(const float* __restrict__ seg, int b, int F, int K, float gamma, float beta,
                                         int normalize, float* __restrict__ out, float* sw) {
  const float* s = seg + (size_t)b * F * K;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    float mx = -INFINITY;
    for (int k = 0; k < K; k++) mx = fmaxf(mx, beta * s[f * K + k]);
    float den = 0.f;
    for (int k = 0; k < K; k++) den += expf(beta * s[f * K + k] - mx);
    for (int k = 0; k < K; k++) {
      const float sv = s[f * K + k];
      const float p = expf(beta * sv - mx) / den;
      float w = pow_like_torch(sv, gamma) * pow_like_torch(p, gamma);
      if (w < 1e-8f) w = 1e-8f;
      sw[f * K + k] = w;
    }
  }
  __syncthreads();
  if (normalize) {
    float* mn = sw + F * K;
    float* mxv = mn + K;
    if (threadIdx.x < K) {
      float lo = INFINITY, hi = -INFINITY;
      for (int f = 0; f < F; f++) {
        lo = fminf(lo, sw[f * K + threadIdx.x]);
        hi = fmaxf(hi, sw[f * K + threadIdx.x]);
      }
      mn[threadIdx.x] = lo;
      mxv[threadIdx.x] = hi;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < F * K; i += blockDim.x) {
      const int k = i % K;
      float v = (sw[i] - mn[k]) / (mxv[k] - mn[k]);
      if (isnan(v)) v = 1e-8f;                      // nan_to_num_(1e-8)
      else if (isinf(v)) v = v > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
      out[(size_t)b * F * K + i] = v;
    }
  } else {
    for (int i = threadIdx.x; i < F * K; i += blockDim.x) out[(size_t)b * F * K + i] = sw[i];
  }
}

// one CTA per item
__global__ void __launch_bounds__(256) osp_kernel(const float* __restrict__ seg, int F, int K, float gamma, float beta,
                                                  int normalize, float* __restrict__ out) {
  extern __shared__ float sw[];   // [F*K] (+ 2*K min/max)
  osp_item(seg, blockIdx.x, F, K, gamma, beta, normalize, out, sw);
}

// one CTA per (item, set): set g's weights of item b go to out + g B F K, from that set's gamma, beta and normalize
__global__ void __launch_bounds__(256) osp_sets_kernel(const float* __restrict__ seg, int F, int K, OspSets sets,
                                                       float* __restrict__ out) {
  extern __shared__ float sw[];   // [F*K] (+ 2*K min/max)
  const int g = blockIdx.y;
  osp_item(seg, blockIdx.x, F, K, sets.gamma[g], sets.beta[g], sets.normalize[g], out + (size_t)g * gridDim.x * F * K, sw);
}

int launch_osp(const float* seg, int B, int F, int K, float gamma, float beta, int normalize, float* out,
               cudaStream_t st) {
  ProfScope _ps("osp", st);
  const size_t smem = ((size_t)F * K + 2 * K) * sizeof(float);
  if (smem > 48 * 1024) {
    set_error("osp: frames*speakers too large");
    return -1;
  }
  osp_kernel<<<B, 256, smem, st>>>(seg, F, K, gamma, beta, normalize, out);
  DG_LAUNCHED();
  return 0;
}

int launch_osp_sets(const float* seg, int B, int F, int K, const OspSets& sets, int G, float* out, cudaStream_t st) {
  ProfScope _ps("osp", st);
  const size_t smem = ((size_t)F * K + 2 * K) * sizeof(float);
  if (smem > 48 * 1024 || G < 1 || G > DG_MAX_OSP_SETS) {
    set_error("osp_sets: frames*speakers too large, or not 1..64 sets");
    return -1;
  }
  osp_sets_kernel<<<dim3(B, G), 256, smem, st>>>(seg, F, K, sets, out);
  DG_LAUNCHED();
  return 0;
}

// ------------------------------------------------------------------------------------ stats_pool
// grid (ceil(C/64), groups); block 256 = 64 channels x 4 frame groups.  A group is up to 4 pool rows
// q0..q0+nq-1 that share one trunk item (the K local speakers of a chunk): x is read once per pass
// for all of them.  Weights are resized on the fly from F to T frames with the host-built tables
// (idx0, idx1, lam1): nearest has lam1 = 0, linear interpolates (F.interpolate semantics).
constexpr int PK = 4;
__global__ void __launch_bounds__(256)
stats_pool_kernel(const float* __restrict__ x, long long item_pitch, int row_pitch, int T, int C, const float* __restrict__ w, int F, int K,
                  int layout /*0: [B,F,K], 1: [N,F]*/, const int* __restrict__ grp_item, const int* __restrict__ grp_q0,
                  const int* __restrict__ grp_nq, const int* __restrict__ idx0, const int* __restrict__ idx1,
                  const float* __restrict__ lam1, float eps, float* __restrict__ pooled) {
  extern __shared__ float sm[];
  float* wr = sm;                    // [T][PK]
  float* red = sm + (size_t)T * PK;  // [4][64][PK]
  __shared__ float v1s[PK], v2s[PK];
  const int g = blockIdx.y;
  int item, q0, nq;
  if (grp_item) {
    item = grp_item[g]; q0 = grp_q0[g]; nq = grp_nq[g];
  } else {  // fused layout: chunks of PK speakers of item g / ceil(K/PK)
    const int per = (K + PK - 1) / PK;
    item = g / per;
    const int k0 = (g - item * per) * PK;
    q0 = item * K + k0;
    nq = K - k0 < PK ? K - k0 : PK;
  }
  const bool weighted = w != nullptr;
  for (int i = threadIdx.x; i < T * PK; i += blockDim.x) {
    const int t = i / PK, j = i - t * PK;
    float v = 0.f;
    if (j < nq) {
      if (!weighted) v = 1.f;
      else {
        const int q = q0 + j;
        const int i0 = idx0[t], i1 = idx1[t];
        const float l1 = lam1[t];
        const size_t base = layout == 0 ? (size_t)(q / K) * F * K + (q % K) : (size_t)q * F;
        const size_t fs = layout == 0 ? K : 1;
        const float a = w[base + i0 * fs];
        v = l1 == 0.f ? a : (1.f - l1) * a + l1 * w[base + i1 * fs];
      }
    }
    wr[i] = v;
  }
  __syncthreads();
  if (threadIdx.x < PK) {
    float s1 = 0.f, s2 = 0.f;
    for (int t = 0; t < T; t++) {
      const float v = wr[t * PK + threadIdx.x];
      s1 += v;
      s2 = fmaf(v, v, s2);
    }
    v1s[threadIdx.x] = s1 + eps;
    v2s[threadIdx.x] = s2;
  }
  const int cl = threadIdx.x & 63, tg = threadIdx.x >> 6;
  const int c = blockIdx.x * 64 + cl;
  const bool ok = c < C;
  const float* xb = x + (size_t)item * item_pitch + c;
  float acc[PK] = {0.f, 0.f, 0.f, 0.f};
  if (ok)
    for (int t = tg; t < T; t += 4) {
      const float xv = xb[(size_t)t * row_pitch];
      const float4 wv = *reinterpret_cast<const float4*>(&wr[t * PK]);
      acc[0] = fmaf(xv, wv.x, acc[0]); acc[1] = fmaf(xv, wv.y, acc[1]);
      acc[2] = fmaf(xv, wv.z, acc[2]); acc[3] = fmaf(xv, wv.w, acc[3]);
    }
#pragma unroll
  for (int j = 0; j < PK; j++) red[(tg * 64 + cl) * PK + j] = acc[j];
  __syncthreads();
  float mean[PK];
#pragma unroll
  for (int j = 0; j < PK; j++) {
    const float s = red[(0 * 64 + cl) * PK + j] + red[(1 * 64 + cl) * PK + j] + red[(2 * 64 + cl) * PK + j] +
                    red[(3 * 64 + cl) * PK + j];
    mean[j] = s / v1s[j];
    acc[j] = 0.f;
  }
  __syncthreads();
  if (ok)
    for (int t = tg; t < T; t += 4) {
      const float xv = xb[(size_t)t * row_pitch];
      const float4 wv = *reinterpret_cast<const float4*>(&wr[t * PK]);
      float d;
      d = xv - mean[0]; acc[0] = fmaf(d * d, wv.x, acc[0]);
      d = xv - mean[1]; acc[1] = fmaf(d * d, wv.y, acc[1]);
      d = xv - mean[2]; acc[2] = fmaf(d * d, wv.z, acc[2]);
      d = xv - mean[3]; acc[3] = fmaf(d * d, wv.w, acc[3]);
    }
#pragma unroll
  for (int j = 0; j < PK; j++) red[(tg * 64 + cl) * PK + j] = acc[j];
  __syncthreads();
  if (tg == 0 && ok) {
    for (int j = 0; j < nq; j++) {
      const float s = red[(0 * 64 + cl) * PK + j] + red[(1 * 64 + cl) * PK + j] + red[(2 * 64 + cl) * PK + j] +
                      red[(3 * 64 + cl) * PK + j];
      float var;
      if (weighted) var = s / (v1s[j] - v2s[j] / v1s[j] + eps);
      else var = s / (float)(T - 1);            // torch.std(unbiased=True)
      float* o = pooled + (size_t)(q0 + j) * 2 * C;
      o[c] = mean[j];
      o[C + c] = sqrtf(var);
    }
  }
}

int launch_stats_pool_ex(const float* x, int stride, int T, int C, const float* w, int F, int K, int layout,
                         int n_groups, const int* grp_item, const int* grp_q0, const int* grp_nq, const int* idx0,
                         const int* idx1, const float* lam1, float eps, float* pooled, cudaStream_t st, long long item_pitch,
                         int row_pitch) {
  ProfScope _ps("stats_pool", st);
  const size_t smem = ((size_t)T * PK + 4 * 64 * PK) * sizeof(float);
  dim3 grid((C + 63) / 64, n_groups);
  if (!item_pitch) item_pitch = (long long)stride * C;       // dense [item][stride rows][C]
  if (!row_pitch) row_pitch = C;
  stats_pool_kernel<<<grid, 256, smem, st>>>(x, item_pitch, row_pitch, T, C, w, F, K, layout, grp_item, grp_q0, grp_nq, idx0, idx1,
                                             lam1, eps, pooled);
  DG_LAUNCHED();
  return 0;
}

int launch_stats_pool(const float* x, int B, int stride, int T, int C, const float* w, int F, int K, const int* idx0,
                      const int* idx1, const float* lam1, float eps, float* pooled, cudaStream_t st, long long item_pitch,
                      int row_pitch) {
  const int per = (K + PK - 1) / PK;
  return launch_stats_pool_ex(x, stride, T, C, w, F, K, 0, B * per, nullptr, nullptr, nullptr, idx0, idx1, lam1, eps,
                              pooled, st, item_pitch, row_pitch);
}

// ------------------------------------------------------------------ fused pooling: weights and finalisation
// Row weights of the fused TDNN5 + pooling epilogue (gemm_tc.cu, TC_POOL): the OSP weights resized from F to T frames exactly
// like stats_pool_kernel does, one float4 per trunk row (zero past the T valid frames of an item / for absent speakers), and
// v1 = sum w (+ eps), v2 = sum w^2 per (item, speaker) in the same summation order as stats_pool_kernel.
// Item b's row weights and weight sums; shared by pool_weights_kernel and pool_weights_sets_kernel.
__device__ __forceinline__ void pool_weights_item(const float* __restrict__ w, int b, int F, int K, int item_rows, int T,
                                                  const int* __restrict__ idx0, const int* __restrict__ idx1,
                                                  const float* __restrict__ lam1, float eps, float* __restrict__ row_w,
                                                  float* __restrict__ vsum, float* wr /*[T][4] shared*/) {
  for (int i = threadIdx.x; i < item_rows * 4; i += blockDim.x) {
    const int t = i >> 2, k = i & 3;
    float v = 0.f;
    if (t < T && k < K) {
      const size_t base = (size_t)b * F * K + k;
      const float a = w[base + (size_t)idx0[t] * K];
      const float l1 = lam1[t];
      v = l1 == 0.f ? a : (1.f - l1) * a + l1 * w[base + (size_t)idx1[t] * K];
    }
    if (t < T) wr[i] = v;
    row_w[((size_t)b * item_rows + t) * 4 + k] = v;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    float s1 = 0.f, s2 = 0.f;
    for (int t = 0; t < T; t++) {
      const float v = wr[t * 4 + threadIdx.x];
      s1 += v;
      s2 = fmaf(v, v, s2);
    }
    vsum[((size_t)b * K + threadIdx.x) * 2] = s1 + eps;
    vsum[((size_t)b * K + threadIdx.x) * 2 + 1] = s2;
  }
}

__global__ void __launch_bounds__(256) pool_weights_kernel(const float* __restrict__ w, int F, int K, int item_rows, int T,
                                                           const int* __restrict__ idx0, const int* __restrict__ idx1,
                                                           const float* __restrict__ lam1, float eps, float* __restrict__ row_w,
                                                           float* __restrict__ vsum) {
  extern __shared__ float wr[];      // [T][4]
  pool_weights_item(w, blockIdx.x, F, K, item_rows, T, idx0, idx1, lam1, eps, row_w, vsum, wr);
}

// one CTA per (item, set): set g reads its OSP weights at w + g B F K and writes its row weights at row_w + g rw_stride and its
// weight sums at vsum + g B K 2
__global__ void __launch_bounds__(256) pool_weights_sets_kernel(const float* __restrict__ w, int F, int K, int item_rows, int T,
                                                                const int* __restrict__ idx0, const int* __restrict__ idx1,
                                                                const float* __restrict__ lam1, float eps,
                                                                float* __restrict__ row_w, long long rw_stride,
                                                                float* __restrict__ vsum) {
  extern __shared__ float wr[];      // [T][4]
  const int g = blockIdx.y;
  const size_t B = gridDim.x;
  pool_weights_item(w + g * B * F * K, blockIdx.x, F, K, item_rows, T, idx0, idx1, lam1, eps, row_w + g * rw_stride,
                    vsum + g * B * K * 2, wr);
}

int launch_pool_weights(const float* w, int B, int F, int K, int item_rows, int T, const int* idx0, const int* idx1,
                        const float* lam1, float eps, float* row_w, float* vsum, cudaStream_t st) {
  ProfScope _ps("pool_weights", st);
  pool_weights_kernel<<<B, 256, (size_t)T * 4 * sizeof(float), st>>>(w, F, K, item_rows, T, idx0, idx1, lam1, eps, row_w, vsum);
  DG_LAUNCHED();
  return 0;
}

int launch_pool_weights_sets(const float* w, int B, int G, int F, int K, int item_rows, int T, const int* idx0, const int* idx1,
                             const float* lam1, float eps, float* row_w, long long rw_stride, float* vsum, cudaStream_t st) {
  ProfScope _ps("pool_weights", st);
  pool_weights_sets_kernel<<<dim3(B, G), 256, (size_t)T * 4 * sizeof(float), st>>>(w, F, K, item_rows, T, idx0, idx1, lam1, eps,
                                                                                 row_w, rw_stride, vsum);
  DG_LAUNCHED();
  return 0;
}

// pyannote StatsPool from the partial sums of the fused epilogue (d = x - pivot, pivot = the BatchNorm shift):
//   mean = sum(w x) / v1,  std = sqrt( sum(w (x - mean)^2) / (v1 - v2 / v1 + eps) ),  v1 = sum w + eps, v2 = sum w^2,
// v1, v2 as launch_pool_weights sums them (one near-one-hot speaker makes v1 - v2 / v1 a cancellation whose rounding must match
// the un-fused pooling's).  Tile t of the item holds S1_t = sum w e, S2_t = sum w e^2 of e = d - p_t around its own pivot p_t
// (a value of the channel).  In double, in tile order, each tile is shifted to the pivot P of the item's first tile,
//   sum w (d - P) += S1_t + W_t (p_t - P),  sum w (d - P)^2 += S2_t + 2 (p_t - P) S1_t + W_t (p_t - P)^2,
// with W_t = sum w over the tile's rows (from the row weights, once per (item, speaker)).  Every term is of the size of the
// channel's spread, so a channel whose mean is large next to its spread loses nothing to cancellation.
constexpr int POOL_FIN_TILES = 32;   // tile weights staged per round
__global__ void __launch_bounds__(128) pool_finalize_kernel(const float* __restrict__ part, const float* __restrict__ row_w,
                                                            const float* __restrict__ vsum, const float* __restrict__ pivot, int K,
                                                            int C, int item_rows, int T, float eps, float* __restrict__ pooled) {
  __shared__ double wt[POOL_FIN_TILES];
  const int q = blockIdx.y, b = q / K, k = q - b * K;
  const int c = blockIdx.x * blockDim.x + threadIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = (long long)b * item_rows, r1 = r0 + T - 1, mt_lo = r0 / 128;
  const int ntiles = (int)(r1 / 128 - mt_lo + 1);
  auto slots = [&](long long mt) { return part + (((size_t)mt * 2 + (int)(b - (mt * 128) / item_rows)) * TC_POOL_SLOTS) * C + c; };
  const double P = c < C ? slots(mt_lo)[8 * C] : 0.0;
  double W = 0, s1 = 0, s2 = 0, s2c = 0;
  for (int t0 = 0; t0 < ntiles; t0 += POOL_FIN_TILES) {
    const int nt = min(POOL_FIN_TILES, ntiles - t0);
    if (t0) __syncthreads();                // the previous round's weights are read
    // the item's weight in each tile (rows past T carry weight 0): warp w sums tiles w, w + 4, ..., a fixed shuffle tree
    for (int t = warp; t < nt; t += 4) {
      const long long mt = mt_lo + t0 + t;
      double sw = 0;
      for (long long r = max(r0, mt * 128) + lane; r <= min(r1, mt * 128 + 127); r += 32) sw += row_w[r * 4 + k];
      for (int o = 16; o > 0; o >>= 1) sw += __shfl_xor_sync(0xffffffffu, sw, o);
      if (lane == 0) wt[t] = sw;
    }
    __syncthreads();
    if (c < C)
      for (int t = 0; t < nt; t++) {
        const float* p = slots(mt_lo + t0 + t);
        const double w = wt[t], a1 = p[2 * k * C], a2 = p[(2 * k + 1) * C], dp = (double)p[8 * C] - P;
        W += w;
        s1 += a1 + w * dp;
        s2 += a2 + dp * (2.0 * a1 + w * dp);
        s2c += a2;
      }
  }
  if (c >= C) return;
  const double v1 = vsum[(size_t)q * 2], v2 = vsum[(size_t)q * 2 + 1], pv = pivot[c];
  const double dm = (s1 + W * P - pv * (double)eps) / v1, dq = dm - P;     // mean - pivot; mean - P
  double num = s2 - 2.0 * dq * s1 + dq * dq * W;
  // The float32 sums around the pivots leave about 2^-22 of s2c in `num`.  Below 2^-20 s2c the variance is not resolved and
  // is 0: that happens only when the weight sits on frames far from the pivots (one frame carries all the weight: exactly 0
  // over a denominator of 1e-8), which is what the centred two-pass pooling (stats_pool) returns there.
  if (num < s2c * 9.5367431640625e-7 || num < 0) num = 0;
  const double var = num / (v1 - v2 / v1 + (double)eps);
  float* o = pooled + (size_t)q * 2 * C;
  o[c] = (float)(pv + dm);
  o[C + c] = (float)sqrt(var);
}

int launch_pool_finalize(const float* part, const float* row_w, const float* vsum, const float* pivot, int B, int K, int C,
                         int item_rows, int T, float eps, float* pooled, cudaStream_t st) {
  ProfScope _ps("pool_finalize", st);
  dim3 grid((C + 127) / 128, B * K);
  pool_finalize_kernel<<<grid, 128, 0, st>>>(part, row_w, vsum, pivot, K, C, item_rows, T, eps, pooled);
  DG_LAUNCHED();
  return 0;
}

// ---------------------------------------------------------------------------------------- l2norm
__global__ void __launch_bounds__(256) l2norm_kernel(const float* __restrict__ in, int rows, int D, float norm,
                                                     float* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* e = in + (size_t)row * D;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s = fmaf(e[i], e[i], s);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float n = sqrtf(s);
  for (int i = lane; i < D; i += 32) out[(size_t)row * D + i] = norm * e[i] / n;
}

int launch_l2norm(const float* in, int rows, int D, float norm, float* out, cudaStream_t st) {
  ProfScope _ps("l2norm", st);
  l2norm_kernel<<<(rows + 7) / 8, 256, 0, st>>>(in, rows, D, norm, out);
  DG_LAUNCHED();
  return 0;
}

// ----------------------------------------------------------------------- row flags / row gather
// flags[i] = 1 iff waveform row i is bit-identical to row i-1 (i >= 1)
__global__ void __launch_bounds__(256) row_equal_kernel(const float* __restrict__ wav, int S, int* __restrict__ flags) {
  const int i = blockIdx.x;
  if (i == 0) {
    if (threadIdx.x == 0) flags[0] = 0;
    return;
  }
  const uint32_t* a = reinterpret_cast<const uint32_t*>(wav + (size_t)i * S);
  const uint32_t* b = reinterpret_cast<const uint32_t*>(wav + (size_t)(i - 1) * S);
  int diff = 0;
  for (int k = threadIdx.x; k < S; k += blockDim.x) diff |= (a[k] != b[k]);
  diff = __syncthreads_or(diff);
  if (threadIdx.x == 0) flags[i] = diff ? 0 : 1;
}

int launch_row_equal_flags(const float* wav, int N, int S, int* flags, cudaStream_t st) {
  row_equal_kernel<<<N, 256, 0, st>>>(wav, S, flags);
  DG_LAUNCHED();
  return 0;
}

__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, const int* __restrict__ index,
                                                          int cols, float* __restrict__ dst) {
  const float* s = src + (size_t)index[blockIdx.x] * cols;
  float* d = dst + (size_t)blockIdx.x * cols;
  for (int k = threadIdx.x; k < cols; k += blockDim.x) d[k] = s[k];
}

int launch_gather_rows(const float* src, const int* index, int rows, int cols, float* dst, cudaStream_t st) {
  gather_rows_kernel<<<rows, 256, 0, st>>>(src, index, cols, dst);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

// The per-frame Hamming aggregation of the device post-path (DelayedAggregation, reference aggregation.py:73-92,120-218),
// shared by post_chunk (post.cu) and the speech curves of vad.cu.
#pragma once
#include "dg_common.cuh"

namespace dg {

// The speech score of one frame, s [K] (reference vad.py:145-148, torch.amax over the local speakers): the max in float32, and
// a NaN, once taken, is never replaced (x > NaN is false), as torch propagates it.
__device__ __forceinline__ float speaker_max(const float* s, int K) {
  float m = s[0];
  for (int k = 1; k < K; k++) {
    const float x = s[k];
    m = (x > m || isnan(x)) ? x : m;
  }
  return m;
}

// Output frame fo of a chunk whose plan row is pl ([0] nb, [1] nf, [2] first_nf, [3] first_lo, [4 ..] lo per buffer, see
// post.cu), nfo = first_nf > 0 ? first_nf : nf.  val(j, idx) is the score of buffer j (oldest first) at frame idx, as a double.
// The prepended part of the very first buffer is its raw score; everything else is
//   sum_j hamming[idx_j] * val(j, idx_j) / sum_j hamming[idx_j]
// over edge-clamped crops, in float64 with every operation rounded on its own (numpy's order, no fused multiply-add).
template <class Val>
__device__ __forceinline__ double post_frame(const int32_t* pl, int nb, int nf, int nfo, int first_lo, int F,
                                             const double* __restrict__ hamming, int fo, Val val) {
  const int fa = fo - (nfo - nf);          // frame of the aggregated part
  if (fa < 0) {                             // prepended part of the very first buffer: raw permuted scores
    int idx = first_lo + fo;
    idx = idx < 0 ? 0 : (idx > F - 1 ? F - 1 : idx);
    return val(0, idx);
  }
  double num = 0.0, den = 0.0;
  for (int j = 0; j < nb; j++) {
    int idx = pl[4 + j] + fa;
    idx = idx < 0 ? 0 : (idx > F - 1 ? F - 1 : idx);    // `fixed` crops are edge-padded
    const double v = val(j, idx);
    const double h = hamming[idx];
    const double p = __dmul_rn(h, v);
    num = j ? __dadd_rn(num, p) : p;
    den = j ? __dadd_rn(den, h) : h;
  }
  return __ddiv_rn(num, den);
}

}  // namespace dg

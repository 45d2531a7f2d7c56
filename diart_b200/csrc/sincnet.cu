// SincNet front end (shared by the segmentation and the embedding net, separate weights): the waveform statistics of
// InstanceNorm1d(1, affine) and the per-(item, channel) InstanceNorm statistics that the next layer applies on load.
// The convolutions themselves run on the tensor cores (sinc_tc.cu, gemm_tc.cu).
// Restates pyannote.audio's SincNet.forward (SURVEY.md Appendix A.2); reached from the reference
// through src/diart/models.py:131-133.
#include "dg_common.cuh"

namespace dg {

// ---------------------------------------------------------------------------------------------
// waveform statistics: mean and 1/sqrt(biased var + 1e-5) per item.  One CTA per item, two passes
// (the second one hits L1/L2), per-thread float partials combined in double.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum_d(double v, double* sm) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sm[w] = v;
  __syncthreads();
  double t = 0;
  for (int i = 0; i < nw; i++) t += sm[i];
  return t;
}

__global__ void __launch_bounds__(512) wave_stats_kernel(const float* __restrict__ wav, int S, float* __restrict__ mean,
                                                         float* __restrict__ rstd, const int* __restrict__ skip_flag) {
  if (skip_flag && *skip_flag != 0) return;     // the stream form computes the statistics from per-hop partial sums
  __shared__ double sm[32];
  const float* x = wav + (size_t)blockIdx.x * S;
  float s = 0.f;
  for (int i = threadIdx.x; i < S; i += blockDim.x) s += x[i];
  double m = block_sum_d((double)s, sm) / S;
  float mf = (float)m, q = 0.f;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    float d = x[i] - mf;
    q += d * d;
  }
  double var = block_sum_d((double)q, sm) / S;
  if (threadIdx.x == 0) {
    mean[blockIdx.x] = mf;
    rstd[blockIdx.x] = (float)(1.0 / sqrt(var + 1e-5));
  }
}

int launch_wave_stats(const float* wav, int B, int S, float* mean, float* rstd, cudaStream_t st, const int* skip_flag) {
  ProfScope _ps("wave_stats", st);
  wave_stats_kernel<<<B, 512, 0, st>>>(wav, S, mean, rstd, skip_flag);
  DG_LAUNCHED();
  return 0;
}

// ---- stream form: the B windows are a run of one stream (window b = samples [b*hop, b*hop + S)), so every sample is summed
// ONCE: partial (sum x, sum x^2) per quarter hop in double, then each window adds its 4 S / hop partials.
// (B x S = 82 MB read by 256 CTAs becomes 8.5 MB read by ~1000.)
__global__ void __launch_bounds__(256) stream_sums_kernel(const float* __restrict__ wav, int B, int S, int hop, int sub,
                                                          double* __restrict__ part, const int* __restrict__ flag) {
  if (*flag == 0) return;
  __shared__ double sm[32];
  const long long first = (long long)blockIdx.x * sub;           // first stream sample of this block
  int b = (int)(first / hop);
  if (b > B - 1) b = B - 1;
  const float4* x = reinterpret_cast<const float4*>(wav + (size_t)b * S + (first - (long long)b * hop));
  // sums of x - pivot (the stream's first sample): sum x^2 / S - mean^2 of the raw samples cancels on audio with a DC offset
  const float pv = wav[0];
  float s1 = 0.f, s2 = 0.f;
  for (int i = threadIdx.x; i < (sub >> 2); i += blockDim.x) {
    float4 v = x[i];
    v.x -= pv; v.y -= pv; v.z -= pv; v.w -= pv;
    s1 += (v.x + v.y) + (v.z + v.w);
    s2 = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s2))));
  }
  const double t1 = block_sum_d((double)s1, sm);
  const double t2 = block_sum_d((double)s2, sm);
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = t1;
    part[2 * blockIdx.x + 1] = t2;
  }
}

__global__ void stream_stats_kernel(const float* __restrict__ wav, const double* __restrict__ part, int B, int S, int hop, int sub, float* __restrict__ mean,
                                    float* __restrict__ rstd, const int* __restrict__ flag) {
  if (*flag == 0) return;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int per_hop = hop / sub, n = S / sub;
  double t1 = 0, t2 = 0;
  for (int i = 0; i < n; i++) {
    t1 += part[2 * (b * per_hop + i)];
    t2 += part[2 * (b * per_hop + i) + 1];
  }
  const double m = t1 / S;
  double var = t2 / S - m * m;
  if (var < 0) var = 0;
  mean[b] = (float)((double)wav[0] + m);
  rstd[b] = (float)(1.0 / sqrt(var + 1e-5));
}

bool stream_stats_ok(int S, int hop) { return hop % 16 == 0 && S % (hop / 4) == 0; }
size_t stream_stats_doubles(int B, int S, int hop) { return 2 * ((size_t)(B - 1) * 4 + (size_t)S / (hop / 4)) + 8; }

int launch_stream_stats(const float* wav, int B, int S, int hop, double* part, float* mean, float* rstd, const int* flag,
                        cudaStream_t st) {
  ProfScope _ps("wave_stats", st);
  const int sub = hop / 4;
  const int blocks = (B - 1) * 4 + S / sub;
  stream_sums_kernel<<<blocks, 256, 0, st>>>(wav, B, S, hop, sub, part, flag);
  DG_LAUNCHED();
  stream_stats_kernel<<<(B + 127) / 128, 128, 0, st>>>(wav, part, B, S, hop, sub, mean, rstd, flag);
  DG_LAUNCHED();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// InstanceNorm1d(C, affine) statistics over the T valid rows of each item of x[B, stride, ldc]:
// emits sc = gamma * rstd, sh = beta - mean * gamma * rstd so the consumer computes
// leaky(x * sc + sh) on load.  CTA = (item, 32-channel group); 8 warps stride over rows; sums are
// taken around the first row's value (pivot) to avoid E[x^2]-E[x]^2 cancellation, combined in double.
// ---------------------------------------------------------------------------------------------
// pool != 0: x holds the un-pooled conv output (stride_rows rows per item) and the statistics are taken over
// MaxPool1d(3) of it, i.e. value(t) = max(x[3t], x[3t+1], x[3t+2]) for t < T.
__global__ void __launch_bounds__(256) instnorm_stats_kernel(const float* __restrict__ x, int stride_rows, int T, int C,
                                                             int ldc, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, float* __restrict__ sc,
                                                             float* __restrict__ sh, int pool,
                                                             const int* __restrict__ skip_flag) {
  if (skip_flag && *skip_flag != 0) return;       // the fused stream-form tail produced these statistics
  __shared__ double s1[8][32], s2[8][32];
  const int b = blockIdx.y, c = blockIdx.x * 32 + (threadIdx.x & 31), w = threadIdx.x >> 5;
  const bool ok = c < C;
  const float* xb = x + (size_t)b * stride_rows * ldc;
  auto val = [&](int t) -> float {
    if (!pool) return xb[(size_t)t * ldc + c];
    const float* p = xb + (size_t)(3 * t) * ldc + c;
    return fmaxf(fmaxf(p[0], p[ldc]), p[2 * ldc]);
  };
  const float pivot = ok ? val(0) : 0.f;
  float a1 = 0.f, a2 = 0.f;
  if (ok)
    for (int t = w; t < T; t += 8) {
      float d = val(t) - pivot;
      a1 += d;
      a2 = fmaf(d, d, a2);
    }
  s1[w][threadIdx.x & 31] = a1;
  s2[w][threadIdx.x & 31] = a2;
  __syncthreads();
  if (w == 0 && ok) {
    double t1 = 0, t2 = 0;
    for (int i = 0; i < 8; i++) {
      t1 += s1[i][threadIdx.x];
      t2 += s2[i][threadIdx.x];
    }
    double m = t1 / T, var = t2 / T - m * m;
    if (var < 0) var = 0;
    double mean = (double)pivot + m;
    float r = (float)(1.0 / sqrt(var + 1e-5));
    float gsc = gamma[c] * r;
    sc[(size_t)b * C + c] = gsc;
    sh[(size_t)b * C + c] = beta[c] - (float)mean * gsc;
  }
}

int launch_instnorm_stats(const float* x, int B, int stride_rows, int T, int C, int ldc, const float* gamma,
                          const float* beta, float* sc, float* sh, cudaStream_t st, int pool, const int* skip_flag) {
  ProfScope _ps("instnorm_stats", st);
  dim3 grid((C + 31) / 32, B);
  instnorm_stats_kernel<<<grid, 256, 0, st>>>(x, stride_rows, T, C, ldc, gamma, beta, sc, sh, pool, skip_flag);
  DG_LAUNCHED();
  return 0;
}

// InstanceNorm1d(affine) scale / shift from the per-tile partial sums of gemm_tc's TC_MAXPOOL3 epilogue (tiles of `tile_rows`
// un-pooled rows, a divisor of the item's rows: slot 0 of the item's own tiles).  Tile i holds, for its n_i pooled frames
// v < T of the item (before the bias), the sums S1_i, S2_i of e = v - p_i and e^2 around its pivot p_i (a value of the channel).
// In double, each tile is shifted to the pivot P of the item's first tile,
//   sum (v - P) += S1_i + n_i (p_i - P),  sum (v - P)^2 += S2_i + 2 (p_i - P) S1_i + n_i (p_i - P)^2,
// every term of the size of the channel's spread: no cancellation against the mean however large it is next to the spread.
__global__ void __launch_bounds__(256) instnorm_finalize_kernel(const float* __restrict__ part, int tiles_per_item, int tile_frames,
                                                                int T, int C, int N, const float* __restrict__ bias,
                                                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                float* __restrict__ sc, float* __restrict__ sh, int ld) {
  // 4 tile groups x 64 channels: the loads of a group are independent, the groups are added in a fixed order
  __shared__ double s1[4][64], s2[4][64];
  const int b = blockIdx.x, c = threadIdx.x & 63, grp = threadIdx.x >> 6;
  const long long mt0 = (long long)b * tiles_per_item;
  const int per = (tiles_per_item + 3) / 4, lo = grp * per, hi = min(tiles_per_item, lo + per);
  auto slot = [&](int i, int j) { return (double)part[(((mt0 + i) * 2 + 0) * TC_POOL3_SLOTS + j) * N + c]; };
  const double P = c < C ? slot(0, 2) : 0.0;
  double t1 = 0, t2 = 0;
  if (c < C)
    for (int i = lo; i < hi; i++) {
      const double n = max(0, min(tile_frames, T - i * tile_frames)), a1 = slot(i, 0), dp = slot(i, 2) - P;
      t1 += a1 + n * dp;
      t2 += slot(i, 1) + dp * (2.0 * a1 + n * dp);
    }
  s1[grp][c] = t1;
  s2[grp][c] = t2;
  __syncthreads();
  if (grp != 0 || c >= C) return;
  t1 = ((s1[0][c] + s1[1][c]) + s1[2][c]) + s1[3][c];
  t2 = ((s2[0][c] + s2[1][c]) + s2[2][c]) + s2[3][c];
  const double m = t1 / T;
  double var = t2 / T - m * m;
  if (var < 0) var = 0;
  const double mean = P + m + (double)bias[c];
  const float r = (float)(1.0 / sqrt(var + 1e-5));
  const float gsc = gamma[c] * r;
  sc[(size_t)b * ld + c] = gsc;
  sh[(size_t)b * ld + c] = beta[c] - (float)mean * gsc;
}

int launch_instnorm_finalize(const float* part, int B, int item_rows, int tile_rows, int T, int C, int N, const float* bias,
                             const float* gamma, const float* beta, float* sc, float* sh, int ld, cudaStream_t st) {
  ProfScope _ps("instnorm_finalize", st);
  if (C > 64 || tile_rows < 3 || tile_rows % 3 || item_rows % tile_rows) {
    set_error("instnorm_finalize: at most 64 channels, tiles of whole pooling windows must divide the item");
    return -1;
  }
  instnorm_finalize_kernel<<<B, 256, 0, st>>>(part, item_rows / tile_rows, tile_rows / 3, T, C, N, bias, gamma, beta, sc, sh, ld);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

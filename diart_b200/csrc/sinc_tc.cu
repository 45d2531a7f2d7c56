// SincNet stage 0 on the tensor cores:  InstanceNorm1d(1) -> ParamSincFB (80 x k251, stride 10) -> |.| ->
// MaxPool1d(3)   (pyannote SincNet, SURVEY.md Appendix A.1/A.2; reached through reference models.py:131-133)
//
// As a GEMM the layer is out[t, f] = sum_k x[10 t + k] h[f, k]: M = 7975 conv positions per chunk, N = 80,
// K = 251 (padded to 256), and its A operand is a Toeplitz view of the waveform whose rows OVERLAP (row t
// starts 10 samples = 20 bytes after row t-1).  Instead of materialising a 2 GB im2col matrix per batch, the
// rows are read in place by TMA through tensor maps whose row pitch (240 B) is smaller than the row length:
//
//   * conv positions are split into 12 classes s = t mod 12 (12 = lcm(4, 3)): inside a class consecutive rows
//     are 120 samples = 240 B apart, a legal (16 B multiple) TMA stride;
//   * row (t'', s) starts at sample 120 t'' + 10 s, i.e. at byte offset 20 s mod 16 in {0, 4, 8, 12}: the
//     normalised waveform is stored as four copies shifted by 0/2/4/6 samples so that class s reads copy
//     s mod 4 at an 8-sample-aligned inner coordinate e_s = 10 s - 2 (s mod 4);
//   * the three classes 3q, 3q+1, 3q+2 of a MaxPool group are three accumulators of ONE CTA tile, so the
//     pooled value is an element-wise max over accumulators in the epilogue: pooled row p = 4 t'' + q.
//   * items are laid out back to back with 667 rows each, so 128-row tiles run across item boundaries
//     (rows 665/666 of an item are padding that the epilogue drops).
//
// hi/lo split precision as in gemm_tc.cu.  CTA = 288 threads: warp 8 TMA producer (A tiles, 3-stage ring; the 80 KB
// filter bank hi/lo is loaded once and stays resident), warps 0-7 two warpgroups, one per 64-row half of the tile, each
// with the three class accumulators (3 x m64n80 wgmma, float32 in registers) and the epilogue straight from the registers.
#include <stdlib.h>
#include <string.h>

#include "dg_common.cuh"
#include "tc_ptx.cuh"

namespace dg {

constexpr int ST_ROWS = 128, ST_N = 80, ST_KB = 4, ST_NSTAGE = 3, ST_WP = 2;   // 2 filter planes: hi, lo
constexpr int ST_A_BYTES = ST_ROWS * 64 * 2;           // 16 KB per plane per k-block
constexpr int ST_STAGE = 2 * ST_A_BYTES;               // hi + lo
constexpr int ST_W_BYTES = ST_N * 64 * 2;              // 10 KB per plane per k-block
constexpr int ST_W_TOTAL = ST_KB * ST_WP * ST_W_BYTES; // 80 KB
constexpr int ST_SMEM = ST_W_TOTAL + ST_NSTAGE * ST_STAGE + 256 + 1024;
constexpr int ST_THREADS = 288;

struct SincTcMaps {
  CUtensorMap a_hi[4], a_lo[4];   // shifted copies of the normalised waveform, hi / lo planes
  CUtensorMap w[ST_WP];           // filter bank [80][256]: fp16 hi and lo planes
};

__global__ void __launch_bounds__(ST_THREADS, 1)
sinc0_tc_kernel(const __grid_constant__ SincTcMaps maps, int row_tiles, int rows_total, int rows_per_item, int T0,
                int S0, float* __restrict__ p0, float gamma, const float* __restrict__ cf,
                float* __restrict__ craw, int P, const int* __restrict__ flag, int want) {
  // stream form (see the end of this file): the per-window launch and the stream launch are both enqueued and a device
  // flag -- "the batch is a run of overlapping windows of one stream" -- decides which of the two does the work
  if (flag && ((*flag != 0) != (want != 0))) return;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* wsm = smem;                       // [kb][plane][80 x 128 B]
  unsigned char* asm_ = smem + ST_W_TOTAL;         // [stage][plane][128 x 128 B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ST_W_TOTAL + ST_NSTAGE * ST_STAGE);
  uint64_t* full = bars;
  uint64_t* empty = bars + ST_NSTAGE;
  uint64_t* w_full = bars + 2 * ST_NSTAGE;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform
  const int num_tiles = row_tiles * 4;

  if (threadIdx.x == 0) {
    for (int s = 0; s < ST_NSTAGE; s++) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);     // one arrival per consumer warpgroup
    }
    mbar_init(w_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(w_full, ST_W_TOTAL);
      for (int kb = 0; kb < ST_KB; kb++) {
        for (int pl = 0; pl < ST_WP; pl++)
          tma_load_2d(wsm + (kb * ST_WP + pl) * ST_W_BYTES, &maps.w[pl], kb * 64, 0, w_full);
      }
      int stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int rt = tile >> 2, q = tile & 3;
        for (int kb = 0; kb < ST_KB; kb++)
          for (int s3 = 0; s3 < 3; s3++) {
            const int s = 3 * q + s3, c = s & 3, e = 10 * s - 2 * c;
            mbar_wait(&empty[stage], phase ^ 1);
            unsigned char* st = asm_ + stage * ST_STAGE;
            mbar_expect_tx(&full[stage], ST_STAGE);
            tma_load_2d(st, &maps.a_hi[c], e + kb * 64, rt * ST_ROWS, &full[stage]);
            tma_load_2d(st + ST_A_BYTES, &maps.a_lo[c], e + kb * 64, rt * ST_ROWS, &full[stage]);
            if (++stage == ST_NSTAGE) {
              stage = 0;
              phase ^= 1;
            }
          }
      }
    }
    return;
  }
  // ===================================================================== MMA + epilogue (warps 0..7)
  const int wg = warp >> 2, wq = warp & 3;
  const bool signal = (threadIdx.x & 127) == 0;
  mbar_wait(w_full, 0);
  int stage = 0, phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int rt = tile >> 2, q = tile & 3;
    float acc[3][ST_N / 2];
    int prev = -1;
    for (int kb = 0; kb < ST_KB; kb++) {
      const uint32_t wa = smem_u32(wsm + kb * ST_WP * ST_W_BYTES);
      const uint64_t w_hi = wg_desc(wa), w_lo = wg_desc(wa + ST_W_BYTES);
#pragma unroll
      for (int s3 = 0; s3 < 3; s3++) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(asm_ + stage * ST_STAGE) + wg * (64 * 128);   // this warpgroup's 64 rows
        const uint64_t a_hi = wg_desc(sa), a_lo = wg_desc(sa + ST_A_BYTES);
        wg_fence_acc(acc[s3]);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
          const uint64_t adv = (uint64_t)((ks * 32) >> 4);
          // hi + lo carry 22 significand bits of both operands: three products
          wgmma_ss<ST_N>(acc[s3], a_lo + adv, w_hi + adv, (kb | ks) != 0);
          wgmma_ss<ST_N>(acc[s3], a_hi + adv, w_lo + adv, 1);
          wgmma_ss<ST_N>(acc[s3], a_hi + adv, w_hi + adv, 1);
        }
        wg_commit();
        wg_wait<1>();
        wg_fence_acc(acc[s3]);
        if (prev >= 0 && signal) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == ST_NSTAGE) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    wg_wait<0>();
#pragma unroll
    for (int s3 = 0; s3 < 3; s3++) wg_fence_acc(acc[s3]);
    if (signal) mbar_arrive(&empty[prev]);
    // thread rows: 64 wg + 16 wq + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
#pragma unroll
    for (int hr = 0; hr < 2; hr++) {
      const int R = rt * ST_ROWS + 64 * wg + 16 * wq + (lane >> 2) + 8 * hr;   // flattened (item, t'') row
      if (craw) {
        // stream form: the raw convolution outputs of the three classes, conv position 12 t'' + 3 q + j
        const long long pos0 = 12LL * R + 3 * q;
#pragma unroll
        for (int j3 = 0; j3 < 3; j3++)
          if (R < rows_total && pos0 + j3 < P) {
            float* o2 = craw + (size_t)(pos0 + j3) * ST_N + 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < ST_N / 8; j++)
              *reinterpret_cast<float2*>(o2 + 8 * j) = make_float2(acc[j3][4 * j + 2 * hr], acc[j3][4 * j + 2 * hr + 1]);
          }
      } else {
        const int b = R / rows_per_item, tpp = R - b * rows_per_item;
        const int p = 4 * tpp + q;                               // pooled output row
        if (R < rows_total && p < T0) {
          float* o = p0 + ((size_t)b * S0 + p) * ST_N + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < ST_N / 8; j++) {
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
              // the planes hold the standardised waveform; InstanceNorm1d(1)'s affine enters here:
              // conv(gamma * x + beta) = gamma * conv(x) + beta * sum_k h[k]
              const int i = 4 * j + 2 * hr + e;
              const float c0 = cf[8 * j + 2 * (lane & 3) + e];
              v[e] = fmaxf(fmaxf(fabsf(fmaf(gamma, acc[0][i], c0)), fabsf(fmaf(gamma, acc[1][i], c0))),
                           fabsf(fmaf(gamma, acc[2][i], c0)));
            }
            *reinterpret_cast<float2*>(o + 8 * j) = make_float2(v[0], v[1]);
          }
        }
      }
    }
  }
}

// normalised waveform -> four shifted copies, fp16 hi / lo planes:  plane[c][b*Lp + i] = split(xn[b][i + 2c])
__global__ void __launch_bounds__(256) sinc_prep_kernel(const float* __restrict__ wav, const float* __restrict__ mean,
                                                        const float* __restrict__ rstd, int S, int Lp, size_t plane_elems,
                                                        uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                                        const int* __restrict__ skip_flag) {
  if (skip_flag && *skip_flag != 0) return;     // the stream form does the work
  const int b = blockIdx.y;
  const float mu = mean[b], sc = rstd[b];
  const float* x = wav + (size_t)b * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Lp + 8; i += gridDim.x * blockDim.x) {
    const float v = i < S ? (x[i] - mu) * sc : 0.f;            // standardised waveform; the affine is applied in sinc0's epilogue
    uint16_t h, l;
    split_h16(v, h, l);
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int j = i - 2 * c;                                 // copy c holds xn[j + 2c] at position j
      if (j >= 0 && j < Lp) {
        hi[(size_t)c * plane_elems + (size_t)b * Lp + j] = h;
        lo[(size_t)c * plane_elems + (size_t)b * Lp + j] = l;
      }
    }
  }
}

static int make_map2(CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint64_t pitch_bytes,
                     uint32_t box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return -2;
  }
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (overlapping-row waveform view) failed with code " + std::to_string((int)r));
    return -2;
  }
  return 0;
}

int sinc_tc_rows_per_item(const Geom& g) {
  const int by_rows = (g.T0c + 11) / 12, by_len = (g.S + 8 + 119) / 120;
  return by_rows > by_len ? by_rows : by_len;
}
size_t sinc_tc_plane_elems(int B, const Geom& g) { return (size_t)B * sinc_tc_rows_per_item(g) * 120 + 1024; }

// filt [251][80] float32 (k-major) -> two fp16 planes [2][80][256] (n-major, K padded with zeros):
// hi = rn16(w), lo = rn16(w - hi)
void sinc_tc_pack_filters(const float* filt, uint16_t* planes) {
  static float w[80 * 256];
  memset(w, 0, sizeof(w));
  for (int k = 0; k < 251; k++)
    for (int f = 0; f < 80; f++) w[f * 256 + k] = filt[k * 80 + f];
  split_weights_host(w, 80, 80, 256, planes, planes + 80 * 256);
}

// per-filter constant of the folded InstanceNorm1d(1) affine: cf[f] = beta * sum_k h[f][k]
void sinc_tc_affine_consts(const float* filt /*[251][80]*/, float beta, float* cf /*[80]*/) {
  for (int f = 0; f < 80; f++) {
    double s = 0;
    for (int k = 0; k < 251; k++) s += filt[k * 80 + f];
    cf[f] = (float)(beta * s);
  }
}

// standardised waveform -> four shifted fp16 hi/lo copies (shared by every SincNet that reads this batch)
int launch_sinc_prep(const float* wav, const float* mean, const float* rstd, int B, const Geom& g, void* planes_hi,
                     void* planes_lo, cudaStream_t st, const int* skip_flag) {
  const int rpi = sinc_tc_rows_per_item(g), Lp = rpi * 120;
  const size_t plane = sinc_tc_plane_elems(B, g);
  ProfScope _ps("sinc0_prep", st);
  // (grid-stride in x: about 2048 CTAs in all -- this launch usually returns at once on the stream-form flag, and 80 k
  // empty CTAs cost 45 us)
  const int want_x = (2048 + B - 1) / B, max_x = (Lp + 8 + 255) / 256;
  dim3 grid(want_x < max_x ? want_x : max_x, B);
  sinc_prep_kernel<<<grid, 256, 0, st>>>(wav, mean, rstd, g.S, Lp, plane, reinterpret_cast<uint16_t*>(planes_hi),
                                         reinterpret_cast<uint16_t*>(planes_lo), skip_flag);
  DG_LAUNCHED();
  return 0;
}

static int sinc0_launch_common(const void* w_planes, uint64_t rows, int rpi, size_t plane, const void* planes_hi,
                               const void* planes_lo, int T0, int S0, float* p0, float gamma, const float* cf_dev, float* craw,
                               int P, const int* flag, int want, cudaStream_t st) {
  SincTcMaps maps;
  for (int c = 0; c < 4; c++) {
    const __nv_bfloat16* bh = reinterpret_cast<const __nv_bfloat16*>(planes_hi) + (size_t)c * plane;
    const __nv_bfloat16* bl = reinterpret_cast<const __nv_bfloat16*>(planes_lo) + (size_t)c * plane;
    if (make_map2(&maps.a_hi[c], bh, 384, rows, 240, ST_ROWS) || make_map2(&maps.a_lo[c], bl, 384, rows, 240, ST_ROWS))
      return -2;
  }
  for (int pl = 0; pl < ST_WP; pl++)
    if (make_map2(&maps.w[pl], reinterpret_cast<const uint16_t*>(w_planes) + (size_t)pl * 80 * 256, 256, 80, 512, ST_N))
      return -2;
  auto kern = sinc0_tc_kernel;
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done)) DG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_SMEM));
  const int sms = usable_sms();
  const int row_tiles = (int)((rows + ST_ROWS - 1) / ST_ROWS);
  const int tiles = row_tiles * 4;
  kern<<<tiles < sms ? tiles : sms, ST_THREADS, ST_SMEM, st>>>(maps, row_tiles, (int)rows, rpi, T0, S0, p0, gamma, cf_dev, craw, P,
                                                              flag, want);
  DG_LAUNCHED();
  return 0;
}

// `skip_flag` (device, nullable): when it is non-zero the stream form below produces p0 and this launch returns at once
int launch_sinc0_tc(float gamma, const float* cf_dev, const void* w_planes, int B, const Geom& g, const void* planes_hi,
                    const void* planes_lo, float* p0, cudaStream_t st, const int* skip_flag) {
  const int rpi = sinc_tc_rows_per_item(g);
  ProfScope _ps("sinc0", st);
  return sinc0_launch_common(w_planes, (uint64_t)B * rpi, rpi, sinc_tc_plane_elems(B, g), planes_hi, planes_lo, g.T0, g.S0, p0,
                             gamma, cf_dev, nullptr, 0, skip_flag, 0, st);
}

// ---------------------------------------------------------------------------------------------------------------------
// Stream form.  The batches of the hot path are runs of 90 %-overlapping windows of ONE audio stream (window b = samples
// [b*hop, b*hop + S), reference src/diart/operators.py:44-100), and the sinc layer is the only one before the first
// per-window normalisation.  Because InstanceNorm1d(1) is an affine map per window,
//     conv((x - mu_b) * rstd_b * gamma + beta)[t, f] = gamma * rstd_b * conv(x)[t, f] + (beta - gamma * rstd_b * mu_b) * sum_k h[f, k],
// the convolution of the RAW stream is shared by every window that contains the sample: it is computed once over the
// (B-1)*hop + S unique samples (9.6x fewer conv positions at B = 256) and a streaming kernel applies the per-window
// affine, |.| and MaxPool1d(3) from the L2-resident result.  A device-side bit comparison of the overlapping parts
// (`overlap_check`) decides per batch whether this form or the per-window form runs, so arbitrary batches stay exact.
__global__ void __launch_bounds__(256) overlap_check_kernel(const float* __restrict__ wav, int S, int hop, int* flag) {
  const int b = blockIdx.y, n4 = (S - hop) >> 2;
  const uint4* a = reinterpret_cast<const uint4*>(wav + (size_t)b * S + hop);
  const uint4* c = reinterpret_cast<const uint4*>(wav + (size_t)(b + 1) * S);
  bool bad = false;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    const uint4 x = a[i], y = c[i];
    bad |= (x.x != y.x) | (x.y != y.y) | (x.z != y.z) | (x.w != y.w);
  }
  if (bad) *flag = 0;
}

int launch_overlap_check(const float* wav, int B, int S, int hop, int* flag, cudaStream_t st) {
  ProfScope _ps("overlap_check", st);
  DG_CUDA(cudaMemsetAsync(flag, 1, sizeof(int), st));       // non-zero = "overlapping run"; cleared on the first mismatch
  dim3 grid(8, B - 1);
  overlap_check_kernel<<<grid, 256, 0, st>>>(wav, S, hop, flag);
  DG_LAUNCHED();
  return 0;
}

SincStreamGeom sinc_stream_geom(int B, const Geom& g, int hop) {
  SincStreamGeom sg;
  sg.Ls = (B - 1) * hop + g.S;
  sg.P = (B - 1) * (hop / 10) + g.T0c;
  const int by_rows = (sg.P + 11) / 12, by_len = (sg.Ls + 8 + 119) / 120;
  sg.rows = by_rows > by_len ? by_rows : by_len;
  sg.plane = (size_t)sg.rows * 120 + 1024;
  return sg;
}

// The fp16 hi / lo planes keep 22 bits of what is split, and the lo plane is subnormal below 2^-14 * 2^11.  The raw sample
// would spend those bits on a DC offset, or lose them at a low level, before the window's mean and deviation are applied.  The
// stream is therefore split as s (x - p): p = its first sample, s = the power of two below the first window's reciprocal
// deviation (<= 256, from the 1e-5 epsilon), which is the precision the per-window form has.  With A = gamma rstd_b,
//     A conv(x) + (beta - A mu_b) sum h  =  (A / s) conv(s (x - p)) + (beta - A (mu_b - p)) sum h.
// p and s are left behind the device flag (flag[1], flag[2] as float) for the pooling kernels.
__device__ __forceinline__ float stream_scale(float rstd0) { return exp2f(floorf(log2f(fmaxf(rstd0, 1.f)))); }

// stream -> four shifted fp16 hi / lo copies:  plane[c][i] = split(s (stream[i + 2c] - p))
__global__ void __launch_bounds__(256) stream_prep_kernel(const float* __restrict__ wav, const float* __restrict__ rstd, int S,
                                                          int hop, int Ls, int Lp, size_t plane_elems,
                                                          uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int* __restrict__ flag) {
  if (*flag == 0) return;
  const float pv = wav[0], sc = stream_scale(rstd[0]);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    reinterpret_cast<float*>(flag)[1] = pv;
    reinterpret_cast<float*>(flag)[2] = sc;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Lp + 8; i += gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < Ls) {
      const int b = i < S ? 0 : (i - S) / hop + 1;          // the window that ends with this sample
      v = sc * (wav[(size_t)b * S + (i - b * hop)] - pv);
    }
    uint16_t h, l;
    split_h16(v, h, l);
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int j = i - 2 * c;
      if (j >= 0 && j < Lp) {
        hi[(size_t)c * plane_elems + j] = h;
        lo[(size_t)c * plane_elems + j] = l;
      }
    }
  }
}

int launch_stream_prep(const float* wav, const float* rstd, int B, const Geom& g, int hop, void* planes_hi, void* planes_lo,
                       int* flag, cudaStream_t st) {
  const SincStreamGeom sg = sinc_stream_geom(B, g, hop);
  ProfScope _ps("sinc0_prep", st);
  const int Lp = sg.rows * 120;
  stream_prep_kernel<<<(Lp + 8 + 255) / 256, 256, 0, st>>>(wav, rstd, g.S, hop, sg.Ls, Lp, sg.plane, reinterpret_cast<uint16_t*>(planes_hi),
                                                          reinterpret_cast<uint16_t*>(planes_lo), flag);
  DG_LAUNCHED();
  return 0;
}

// raw convolution of the stream: craw[P][80]
int launch_sinc0_tc_stream(const void* w_planes, int B, const Geom& g, int hop, const void* planes_hi, const void* planes_lo,
                           float* craw, const int* flag, cudaStream_t st) {
  const SincStreamGeom sg = sinc_stream_geom(B, g, hop);
  ProfScope _ps("sinc0", st);
  return sinc0_launch_common(w_planes, (uint64_t)sg.rows, sg.rows, sg.plane, planes_hi, planes_lo, 0, 0, nullptr, 1.f, nullptr,
                             craw, sg.P, flag, 1, st);
}

// ---- stream form, fused tail: the pooled map p0 is never written.  The raw convolution of the stream (68 MB at B = 256) stays
// in L2; one pass over it accumulates the InstanceNorm1d(80) statistics of p0 = max_j |A_b craw + bias_b| per (window, filter),
// a second pass recomputes p0, applies the normalisation + LeakyReLU and writes the 16-bit hi/lo planes Conv1d(80, 60, 5) reads
// (80-channel rows, no padding).  Replaces sinc0_pool + instnorm_stats + split16 of this layer (218 MB written and 2 x 218 MB
// read back per network and step).
//
// Both passes walk the STREAM, not the windows: a CTA stages SP_R (+2 halo) rows of the raw convolution in shared memory once
// and serves every window that contains them (up to ceil(3 T0 / hop10) + 1 = 11), so each row leaves L2 once per pass instead
// of ten times.  Pool groups of different windows have different phases (hop / 10 is not a multiple of 3): a CTA owns the
// groups whose FIRST row lies in its range.
constexpr int SP_R = 96, SP_GL = 16, SP_THREADS = 20 * SP_GL;
// pivot and scale the stream was split with (stream_prep_kernel)
__device__ __forceinline__ float sp_pivot(const int* flag) { return reinterpret_cast<const float*>(flag)[1]; }
__device__ __forceinline__ float sp_scale(const int* flag) { return reinterpret_cast<const float*>(flag)[2]; }

__device__ __forceinline__ float4 sp_value_sm(const float4* __restrict__ rows /*[SP_R + 2][20]*/, int r, int f4, float A,
                                              const float4& bias) {
  const float4 u0 = rows[r * 20 + f4], u1 = rows[(r + 1) * 20 + f4], u2 = rows[(r + 2) * 20 + f4];
  float4 v;
  v.x = fmaxf(fmaxf(fabsf(fmaf(A, u0.x, bias.x)), fabsf(fmaf(A, u1.x, bias.x))), fabsf(fmaf(A, u2.x, bias.x)));
  v.y = fmaxf(fmaxf(fabsf(fmaf(A, u0.y, bias.y)), fabsf(fmaf(A, u1.y, bias.y))), fabsf(fmaf(A, u2.y, bias.y)));
  v.z = fmaxf(fmaxf(fabsf(fmaf(A, u0.z, bias.z)), fabsf(fmaf(A, u1.z, bias.z))), fabsf(fmaf(A, u2.z, bias.z)));
  v.w = fmaxf(fmaxf(fabsf(fmaf(A, u0.w, bias.w)), fabsf(fmaf(A, u1.w, bias.w))), fabsf(fmaf(A, u2.w, bias.w)));
  return v;
}
__device__ __forceinline__ float4 sp_bias(const float* cf, const float* hsum, int f4, float Am) {
  const float4 c4 = reinterpret_cast<const float4*>(cf)[f4], h4 = reinterpret_cast<const float4*>(hsum)[f4];
  return make_float4(fmaf(-Am, h4.x, c4.x), fmaf(-Am, h4.y, c4.y), fmaf(-Am, h4.z, c4.z), fmaf(-Am, h4.w, c4.w));
}
// rows [r0, r0 + SP_R + 2) of craw -> shared memory (zeros past the end of the stream)
__device__ __forceinline__ void sp_stage(const float* __restrict__ craw, long long r0, long long P, float4* rows) {
  for (int i = threadIdx.x; i < (SP_R + 2) * 20; i += SP_THREADS) {
    const long long r = r0 + i / 20;
    rows[i] = r < P ? reinterpret_cast<const float4*>(craw)[r * 20 + (i % 20)] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
// windows with a pool group starting in [r0, r0 + SP_R): b_lo .. b_hi; groups p_lo .. p_hi of window b
__device__ __forceinline__ void sp_windows(long long r0, int B, int hop10, int T0, int& b_lo, int& b_hi) {
  const long long last_start = 3LL * (T0 - 1);
  long long lo = (r0 - last_start + hop10 - 1) / hop10;        // ceil((r0 - last_start) / hop10) for non-negative results
  if (r0 - last_start <= 0) lo = 0;
  b_lo = (int)lo;
  b_hi = (int)min((long long)B - 1, (r0 + SP_R - 1) / hop10);
}
__device__ __forceinline__ void sp_groups(long long r0, int b, int hop10, int T0, int& p_lo, int& p_hi) {
  const long long off = r0 - (long long)b * hop10;             // block start relative to the window
  p_lo = off <= 0 ? 0 : (int)((off + 2) / 3);
  const long long e = off + SP_R;                              // groups with 3 p < e
  p_hi = (int)min((long long)T0, (e + 2) / 3);
}

// p0[b][0][f] for every window: the pivot of the statistics
__global__ void __launch_bounds__(96) sinc_pool_pivot_kernel(const float* __restrict__ craw, const float* __restrict__ mean,
                                                             const float* __restrict__ rstd, const float* __restrict__ cf,
                                                             const float* __restrict__ hsum, float gamma, int hop10,
                                                             float* __restrict__ pv, const int* __restrict__ flag) {
  if (*flag == 0) return;
  const int b = blockIdx.x, f = threadIdx.x;
  if (f >= ST_N) return;
  const float Ar = gamma * rstd[b], A = Ar / sp_scale(flag), Am = Ar * (mean[b] - sp_pivot(flag));
  const float bias = fmaf(-Am, hsum[f], cf[f]);
  const float* src = craw + (size_t)b * hop10 * ST_N + f;
  pv[(size_t)b * ST_N + f] = fmaxf(fmaxf(fabsf(fmaf(A, src[0], bias)), fabsf(fmaf(A, src[ST_N], bias))), fabsf(fmaf(A, src[2 * ST_N], bias)));
}

// partial sums around the pivot: part[b][j][0 / 1][80], j = CTA index relative to the window's first CTA
__global__ void __launch_bounds__(SP_THREADS) sinc_pool_stats_kernel(const float* __restrict__ craw, long long P,
                                                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                     const float* __restrict__ cf, const float* __restrict__ hsum,
                                                                     float gamma, int B, int hop10, int T0, int npart,
                                                                     const float* __restrict__ pv, float* __restrict__ part,
                                                                     const int* __restrict__ flag) {
  if (*flag == 0) return;
  __shared__ float4 rows[(SP_R + 2) * 20];
  __shared__ float4 r1[SP_GL][20], r2[SP_GL][20];
  const long long r0 = (long long)blockIdx.x * SP_R;
  sp_stage(craw, r0, P, rows);
  const int f4 = threadIdx.x % 20, gl = threadIdx.x / 20;
  int b_lo, b_hi;
  sp_windows(r0, B, hop10, T0, b_lo, b_hi);
  __syncthreads();
  for (int b = b_lo; b <= b_hi; b++) {
    int p_lo, p_hi;
    sp_groups(r0, b, hop10, T0, p_lo, p_hi);
    const float Ar = gamma * rstd[b], A = Ar / sp_scale(flag), Am = Ar * (mean[b] - sp_pivot(flag));
    const float4 bias = sp_bias(cf, hsum, f4, Am);
    const float4 pvv = reinterpret_cast<const float4*>(pv + (size_t)b * ST_N)[f4];
    float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
    for (int p = p_lo + gl; p < p_hi; p += SP_GL) {
      const int r = (int)((long long)b * hop10 + 3LL * p - r0);
      const float4 v = sp_value_sm(rows, r, f4, A, bias);
      const float dx = v.x - pvv.x, dy = v.y - pvv.y, dz = v.z - pvv.z, dw = v.w - pvv.w;
      s1.x += dx; s1.y += dy; s1.z += dz; s1.w += dw;
      s2.x = fmaf(dx, dx, s2.x); s2.y = fmaf(dy, dy, s2.y); s2.z = fmaf(dz, dz, s2.z); s2.w = fmaf(dw, dw, s2.w);
    }
    r1[gl][f4] = s1;
    r2[gl][f4] = s2;
    __syncthreads();
    if (gl == 0) {
      float4 a = r1[0][f4], q = r2[0][f4];
      for (int i = 1; i < SP_GL; i++) {
        a.x += r1[i][f4].x; a.y += r1[i][f4].y; a.z += r1[i][f4].z; a.w += r1[i][f4].w;
        q.x += r2[i][f4].x; q.y += r2[i][f4].y; q.z += r2[i][f4].z; q.w += r2[i][f4].w;
      }
      const int j = (int)(blockIdx.x - ((long long)b * hop10) / SP_R);
      float4* o = reinterpret_cast<float4*>(part + ((size_t)b * npart + j) * 2 * ST_N);
      o[f4] = a;
      o[20 + f4] = q;
    }
    __syncthreads();
  }
}

// InstanceNorm1d(80, affine) scale / shift per (window, filter) from the CTA partials (double, fixed order)
__global__ void __launch_bounds__(96) sinc_pool_finalize_kernel(int hop10, int T0, int npart, const float* __restrict__ pv,
                                                                const float* __restrict__ part, const float* __restrict__ g0,
                                                                const float* __restrict__ b0, float* __restrict__ sc,
                                                                float* __restrict__ sh, const int* __restrict__ flag) {
  if (*flag == 0) return;
  const int b = blockIdx.x, f = threadIdx.x;
  if (f >= ST_N) return;
  const long long w0 = (long long)b * hop10;
  const int nj = (int)((w0 + 3LL * (T0 - 1)) / SP_R - w0 / SP_R) + 1;       // CTAs that own a pool group of this window
  double t1 = 0, t2 = 0;
  for (int i = 0; i < nj; i++) {
    t1 += part[((size_t)b * npart + i) * 2 * ST_N + f];
    t2 += part[((size_t)b * npart + i) * 2 * ST_N + ST_N + f];
  }
  const double m = t1 / T0;
  double var = t2 / T0 - m * m;
  if (var < 0) var = 0;
  const double mu = (double)pv[(size_t)b * ST_N + f] + m;
  const float r = (float)(1.0 / sqrt(var + 1e-5));
  const float gsc = g0[f] * r;
  sc[(size_t)b * ST_N + f] = gsc;
  sh[(size_t)b * ST_N + f] = b0[f] - (float)mu * gsc;
}

// p0 recomputed -> leaky(p0 * sc + sh) -> fp16 hi / lo planes [B * S0][80]
__global__ void __launch_bounds__(SP_THREADS) sinc_pool_split_kernel(const float* __restrict__ craw, long long P,
                                                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                     const float* __restrict__ cf, const float* __restrict__ hsum,
                                                                     float gamma, int B, int hop10, int T0, int S0,
                                                                     const float* __restrict__ sc, const float* __restrict__ sh,
                                                                     uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                                                     const int* __restrict__ flag) {
  if (*flag == 0) return;
  __shared__ float4 rows[(SP_R + 2) * 20];
  const long long r0 = (long long)blockIdx.x * SP_R;
  sp_stage(craw, r0, P, rows);
  const int f4 = threadIdx.x % 20, gl = threadIdx.x / 20;
  int b_lo, b_hi;
  sp_windows(r0, B, hop10, T0, b_lo, b_hi);
  __syncthreads();
  for (int b = b_lo; b <= b_hi; b++) {
    int p_lo, p_hi;
    sp_groups(r0, b, hop10, T0, p_lo, p_hi);
    const float Ar = gamma * rstd[b], A = Ar / sp_scale(flag), Am = Ar * (mean[b] - sp_pivot(flag));
    const float4 bias = sp_bias(cf, hsum, f4, Am);
    const float4 s4 = reinterpret_cast<const float4*>(sc + (size_t)b * ST_N)[f4], h4 = reinterpret_cast<const float4*>(sh + (size_t)b * ST_N)[f4];
    uint2* oh = reinterpret_cast<uint2*>(hi + (size_t)b * S0 * ST_N);
    uint2* ol = reinterpret_cast<uint2*>(lo + (size_t)b * S0 * ST_N);
    for (int p = p_lo + gl; p < p_hi; p += SP_GL) {
      const int r = (int)((long long)b * hop10 + 3LL * p - r0);
      const float4 v = sp_value_sm(rows, r, f4, A, bias);
      uint16_t h0, h1, h2, h3, l0, l1, l2, l3;
      split_h16(leaky(fmaf(v.x, s4.x, h4.x)), h0, l0);
      split_h16(leaky(fmaf(v.y, s4.y, h4.y)), h1, l1);
      split_h16(leaky(fmaf(v.z, s4.z, h4.z)), h2, l2);
      split_h16(leaky(fmaf(v.w, s4.w, h4.w)), h3, l3);
      oh[(size_t)p * 20 + f4] = make_uint2(pack_u16x2(h0, h1), pack_u16x2(h2, h3));
      ol[(size_t)p * 20 + f4] = make_uint2(pack_u16x2(l0, l1), pack_u16x2(l2, l3));
    }
  }
}

static int sp_npart(const Geom& g, int hop) { return (3 * g.T0 + SP_R - 1) / SP_R + 2; }
size_t sinc_pool_part_floats(int B, const Geom& g, int hop) { return (size_t)B * sp_npart(g, hop) * 2 * ST_N + (size_t)B * ST_N; }

int launch_sinc_pool_fused(const float* craw, const float* mean, const float* rstd, const float* cf, const float* hsum, float gamma,
                           int B, const Geom& g, int hop, const float* g0, const float* b0, float* part, float* sc, float* sh,
                           void* planes_hi, void* planes_lo, const int* flag, cudaStream_t st) {
  const SincStreamGeom sg = sinc_stream_geom(B, g, hop);
  const int hop10 = hop / 10, npart = sp_npart(g, hop);
  const long long last = (long long)(B - 1) * hop10 + 3LL * (g.T0 - 1);       // last pool-group start of the stream
  const int blocks = (int)(last / SP_R) + 1;
  float* pv = part + (size_t)B * npart * 2 * ST_N;
  {
    ProfScope _ps("sinc0_pool_stats", st);
    sinc_pool_pivot_kernel<<<B, 96, 0, st>>>(craw, mean, rstd, cf, hsum, gamma, hop10, pv, flag);
    DG_LAUNCHED();
    sinc_pool_stats_kernel<<<blocks, SP_THREADS, 0, st>>>(craw, sg.P, mean, rstd, cf, hsum, gamma, B, hop10, g.T0, npart, pv, part, flag);
    DG_LAUNCHED();
    sinc_pool_finalize_kernel<<<B, 96, 0, st>>>(hop10, g.T0, npart, pv, part, g0, b0, sc, sh, flag);
    DG_LAUNCHED();
  }
  ProfScope _ps("sinc0_pool_split", st);
  sinc_pool_split_kernel<<<blocks, SP_THREADS, 0, st>>>(craw, sg.P, mean, rstd, cf, hsum, gamma, B, hop10, g.T0, g.S0, sc, sh,
                                                        reinterpret_cast<uint16_t*>(planes_hi), reinterpret_cast<uint16_t*>(planes_lo),
                                                        flag);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

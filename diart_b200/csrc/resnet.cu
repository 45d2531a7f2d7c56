// Variant B of the embedding row (SURVEY.md 8(a) A8'): pyannote/wespeaker-voxceleb-resnet34-LM -- the small kernels around
// the tensor-core convolutions.  The reference reaches this network through src/diart/models.py:50,59 (README.md:172-173);
// its arithmetic lives in pyannote.audio's WeSpeakerResNet34 + torchaudio.compliance.kaldi.fbank (restated in oracle/nets.py).
//
//   waveform * 2^15 -> kaldi fbank (25 ms / 10 ms frames, DC removal, pre-emphasis 0.97, Hamming, 512-point power spectrum,
//   80 mel bins, log) -> mean normalisation over time -> Conv2d(1, 32, 3) + BN + ReLU -> 16 BasicBlocks -> TSTP -> Linear
//
// Mapping (prototyped against the oracle on the CPU in oracle/fbank_linear.py and oracle/resnet_gemm_form.py):
//   * every linear step of the fbank before the power spectrum collapses into ONE [514, 400] operator applied to an
//     OVERLAPPING-ROW view of the waveform (row pitch 160 samples): a plain launch of the split-precision wgmma GEMM of
//     gemm_tc.cu (K = 400 padded to 448, N = 514 padded to 640), no frame matrix is ever materialised;
//   * maps are channels-last on a zero-padded grid, [item][w = time + 1][h = mel + 1][C], so that a 3x3 convolution is a
//     shifted-window GEMM whose nine taps are row offsets (dw-1) * Hp + (dh-1) and padding is simply the zeros already in
//     memory (gemm_tc.cu, TC_CONV2D epilogue: BatchNorm affine, residual, ReLU, hi/lo planes of the next layer);
//   * this file: waveform -> 16-bit planes, power spectrum -> mel -> log, the time mean, the one-channel stem convolution.
#include <math.h>

#include <vector>

#include "dg_common.cuh"
#include "tc_ptx.cuh"

namespace dg {

// waveform [B, S] float32 -> hi / lo fp16 planes of s_b (x * 2^15 - p_b), [B * S (+ tail)], and 1 / s_b; one block per item.
// The pair keeps 22 bits of what it is given and saturates at 65504.  Given x * 2^15 (what pyannote feeds kaldi.fbank) it
// spends those bits on a DC offset that the frame operator then has to cancel -- rounded to fp16 pairs the operator does not
// annihilate a constant, so a constant stretch at 0.5 gave bins near -5 instead of the floor log(eps) -- and it clips above
// |x| = 4.  p_b is the midpoint of the item's range and s_b the power of two that puts max |x * 2^15 - p_b| in [2^14, 2^15):
// the operator annihilates constants, so p_b drops out of the spectrum (a constant item splits into exact zeros, and each
// frame sees only its own item's pivot), and fb_mel divides s_b back out before the power spectrum.  A constant stretch
// inside an item (digital silence before speech) is not at p_b: `level` [B][S / 80] receives the value of every 80-sample
// piece that is constant, NaN for the others, and fb_mel gives a frame whose five pieces hold one value the floor, which is
// what DC removal leaves of it in exact arithmetic.
__global__ void __launch_bounds__(1024) fb_planes_kernel(const float* __restrict__ wav, int S, uint16_t* __restrict__ hi,
                                                         uint16_t* __restrict__ lo, float* __restrict__ inv_scale,
                                                         float* __restrict__ level) {
  __shared__ float red_mn[32], red_mx[32];
  __shared__ float piv[2];
  const int b = blockIdx.x, n4 = S >> 2;
  const float4* x = reinterpret_cast<const float4*>(wav + (size_t)b * S);
  float mn = INFINITY, mx = -INFINITY;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const float4 v = x[i];
    mn = fminf(mn, fminf(fminf(v.x, v.y), fminf(v.z, v.w)));
    mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  if (lane == 0) {
    red_mn[warp] = mn;
    red_mx[warp] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < warps; w++) {
      mn = fminf(mn, red_mn[w]);
      mx = fmaxf(mx, red_mx[w]);
    }
    const float p = (0.5f * mn + 0.5f * mx) * 32768.f;          // = the level itself when the item is constant
    const float r = fmaxf(mx * 32768.f - p, p - mn * 32768.f);  // the largest |x * 2^15 - p| of the item, rounded as below
    int e = 0;
    if (r > 0.f) frexpf(r, &e);                                 // r < 2^e
    e = min(max(e, -100), 115);
    piv[0] = p;
    piv[1] = ldexpf(1.f, 15 - e);
    inv_scale[b] = ldexpf(1.f, e - 15);
  }
  __syncthreads();
  const float p = piv[0], s = piv[1];
  uint2* ho = reinterpret_cast<uint2*>(hi + (size_t)b * S);
  uint2* lw = reinterpret_cast<uint2*>(lo + (size_t)b * S);
  const int pieces = S / 80;                                    // one warp per piece: lanes 0..19 hold its 20 float4
  for (int q = warp; q < pieces; q += warps) {
    const int i = q * 20 + lane;
    const float4 v = lane < 20 ? x[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float v0 = __shfl_sync(0xffffffffu, v.x, 0);
    const bool same = lane >= 20 || (v.x == v0 && v.y == v0 && v.z == v0 && v.w == v0);
    const bool flat = __all_sync(0xffffffffu, same);
    if (lane == 0) level[(size_t)b * pieces + q] = flat ? v0 : __int_as_float(0x7fc00000);
    if (lane >= 20) continue;
    uint16_t h0, h1, h2, h3, l0, l1, l2, l3;
    split_h16((v.x * 32768.f - p) * s, h0, l0);
    split_h16((v.y * 32768.f - p) * s, h1, l1);
    split_h16((v.z * 32768.f - p) * s, h2, l2);
    split_h16((v.w * 32768.f - p) * s, h3, l3);
    ho[i] = make_uint2(pack_u16x2(h0, h1), pack_u16x2(h2, h3));
    lw[i] = make_uint2(pack_u16x2(l0, l1), pack_u16x2(l2, l3));
  }
}

int launch_fb_planes(const float* wav, int B, int S, void* hi, void* lo, float* inv_scale, float* level, cudaStream_t st) {
  ProfScope _ps("fbank_planes", st);
  if (S % 80) {
    set_error("fbank: sample count must be a multiple of 80");
    return -1;
  }
  fb_planes_kernel<<<B, 1024, 0, st>>>(wav, S, reinterpret_cast<uint16_t*>(hi), reinterpret_cast<uint16_t*>(lo), inv_scale,
                                       level);
  DG_LAUNCHED();
  return 0;
}

// spectrum rows [B * rows_per_item][ld] (re 0..256 | im 257..513) of item b scaled by s_b -> log mel energies [B][T][80]; one
// warp per frame.  1 / s_b is a power of two, so re / s_b and im / s_b are exact: the eps clamp sees the unscaled energies.
// A frame whose 400 samples are one value (`level`, fb_planes) has no energy: the floor.
__global__ void __launch_bounds__(256) fb_mel_kernel(const float* __restrict__ spec, int ld, int rows_per_item, int T, int B,
                                                     const float* __restrict__ inv_scale, const float* __restrict__ level,
                                                     const float* __restrict__ banks /*[80][257]*/, const int* __restrict__ k_lo,
                                                     const int* __restrict__ k_hi, float* __restrict__ logmel) {
  __shared__ float pw[8][260];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long frame = (long long)blockIdx.x * 8 + warp;
  if (frame >= (long long)B * T) return;
  const int b = (int)(frame / T), t = (int)(frame - (long long)b * T);
  const float* row = spec + ((size_t)b * rows_per_item + t) * ld;
  const float inv = inv_scale[b];
  const float* lv = level + (size_t)b * 2 * rows_per_item + 2 * t;        // frame t = 80-sample pieces 2t .. 2t + 4
  const bool flat = lv[0] == lv[1] && lv[0] == lv[2] && lv[0] == lv[3] && lv[0] == lv[4];     // false on NaN
  for (int k = lane; k < 257; k += 32) {
    const float re = row[k] * inv, im = row[257 + k] * inv;
    pw[warp][k] = re * re + im * im;
  }
  __syncwarp();
  for (int m = lane; m < 80; m += 32) {
    float acc = 0.f;
    const float* bk = banks + m * 257;
    for (int k = k_lo[m]; k < k_hi[m]; k++) acc = fmaf(bk[k], pw[warp][k], acc);
    if (flat) acc = 0.f;
    logmel[(size_t)frame * 80 + m] = logf(fmaxf(acc, 1.1920928955078125e-07f));     // max(mel, float32 eps)
  }
}

int launch_fb_mel(const float* spec, int ld, int rows_per_item, int T, int B, const float* inv_scale, const float* level,
                  const float* banks, const int* k_lo, const int* k_hi, float* logmel, cudaStream_t st) {
  ProfScope _ps("fbank_mel", st);
  const long long frames = (long long)B * T;
  fb_mel_kernel<<<(int)((frames + 7) / 8), 256, 0, st>>>(spec, ld, rows_per_item, T, B, inv_scale, level, banks, k_lo, k_hi,
                                                         logmel);
  DG_LAUNCHED();
  return 0;
}

// per (item, mel bin): mean over the T frames (feats - feats.mean(dim=1), float32 like torch)
__global__ void __launch_bounds__(320) fb_mean_kernel(const float* __restrict__ logmel, int T, float* __restrict__ mean) {
  __shared__ float part[4][80];
  const int b = blockIdx.x, m = threadIdx.x % 80, q = threadIdx.x / 80;       // 4 frame groups x 80 bins
  const float* x = logmel + (size_t)b * T * 80 + m;
  float s = 0.f;
  for (int t = q; t < T; t += 4) s += x[(size_t)t * 80];
  part[q][m] = s;
  __syncthreads();
  if (q == 0) mean[b * 80 + m] = (part[0][m] + part[1][m] + part[2][m] + part[3][m]) / (float)T;
}

int launch_fb_mean(const float* logmel, int B, int T, float* mean, cudaStream_t st) {
  ProfScope _ps("fbank_mean", st);
  fb_mean_kernel<<<B, 320, 0, st>>>(logmel, T, mean);
  DG_LAUNCHED();
  return 0;
}

// stem: Conv2d(1, 32, 3, padding 1) on the mean-normalised [T][80] map + BatchNorm2d + ReLU -> planes of the padded
// [T + 2][82][32] map.  w [32][3 (dh: mel)][3 (dw: time)] as torch stores it; one thread per (w, h) position, 32 channels.
__global__ void __launch_bounds__(256) rn_stem_kernel(const float* __restrict__ logmel, const float* __restrict__ mean, int T,
                                                      const float* __restrict__ w, const float* __restrict__ sc,
                                                      const float* __restrict__ sh, uint16_t* __restrict__ hi,
                                                      uint16_t* __restrict__ lo) {
  __shared__ float ws[32 * 9], ss[32], bs[32];
  for (int i = threadIdx.x; i < 288; i += blockDim.x) ws[i] = w[i];
  if (threadIdx.x < 32) {
    ss[threadIdx.x] = sc[threadIdx.x];
    bs[threadIdx.x] = sh[threadIdx.x];
  }
  __syncthreads();
  const int b = blockIdx.y;
  const int pos = blockIdx.x * blockDim.x + threadIdx.x;
  if (pos >= T * 80) return;
  const int t = pos / 80, f = pos - t * 80;
  const float* x = logmel + (size_t)b * T * 80;
  const float* mu = mean + b * 80;
  float in[3][3];     // [dh][dw]
#pragma unroll
  for (int dh = 0; dh < 3; dh++)
#pragma unroll
    for (int dw = 0; dw < 3; dw++) {
      const int ff = f + dh - 1, tt = t + dw - 1;
      in[dh][dw] = (ff >= 0 && ff < 80 && tt >= 0 && tt < T) ? x[(size_t)tt * 80 + ff] - mu[ff] : 0.f;
    }
  const size_t row = ((size_t)b * (T + 2) + t + 1) * 82 + f + 1;
  uint32_t oh[16], ol[16];
#pragma unroll
  for (int c2 = 0; c2 < 16; c2++) {
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int c = 2 * c2 + e;
      float acc = 0.f;
#pragma unroll
      for (int dh = 0; dh < 3; dh++)
#pragma unroll
        for (int dw = 0; dw < 3; dw++) acc = fmaf(ws[c * 9 + dh * 3 + dw], in[dh][dw], acc);
      v[e] = fmaxf(fmaf(acc, ss[c], bs[c]), 0.f);
    }
    uint16_t h0, l0, h1, l1;
    split_h16(v[0], h0, l0);
    split_h16(v[1], h1, l1);
    oh[c2] = pack_u16x2(h0, h1);
    ol[c2] = pack_u16x2(l0, l1);
  }
  uint4* ph = reinterpret_cast<uint4*>(hi + row * 32);
  uint4* pl = reinterpret_cast<uint4*>(lo + row * 32);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    ph[i] = make_uint4(oh[4 * i], oh[4 * i + 1], oh[4 * i + 2], oh[4 * i + 3]);
    pl[i] = make_uint4(ol[4 * i], ol[4 * i + 1], ol[4 * i + 2], ol[4 * i + 3]);
  }
}

int launch_rn_stem(const float* logmel, const float* mean, int B, int T, const float* w, const float* sc, const float* sh,
                   void* hi, void* lo, cudaStream_t st) {
  ProfScope _ps("resnet_stem", st);
  dim3 grid((T * 80 + 255) / 256, B);
  rn_stem_kernel<<<grid, 256, 0, st>>>(logmel, mean, T, w, sc, sh, reinterpret_cast<uint16_t*>(hi), reinterpret_cast<uint16_t*>(lo));
  DG_LAUNCHED();
  return 0;
}

// ---------------------------------------------------------------------------------------------- host-side constants
// kaldi frame operator (oracle/fbank_linear.py: frame_operator): rows 0..256 real, 257..513 imaginary part of the 512-point
// DFT of hamming * preemphasis(frame - mean(frame)); float64 arithmetic, returned as float32 [514][400]
void fbank_frame_operator(std::vector<float>& op) {
  const int n = 400, padded = 512, nb = padded / 2 + 1;
  std::vector<double> m((size_t)n * n);       // m = diag(window) * pre * dc
  // dc = I - 1/n; pre = I - 0.97 * shift (x[0] - 0.97 x[0] for the first sample: replicate padding)
  // (pre * dc)[j][i] = dc[j][i] - 0.97 * dc[max(j-1,0)][i]
  for (int j = 0; j < n; j++) {
    const double win = 0.54 - 0.46 * cos(2.0 * M_PI * j / (n - 1));
    const int jp = j > 0 ? j - 1 : 0;
    for (int i = 0; i < n; i++) {
      const double dj = (i == j ? 1.0 : 0.0) - 1.0 / n, dp = (i == jp ? 1.0 : 0.0) - 1.0 / n;
      m[(size_t)j * n + i] = win * (dj - 0.97 * dp);
    }
  }
  op.assign((size_t)2 * nb * n, 0.f);
  std::vector<double> cs(padded), sn(padded);
  for (int k = 0; k < padded; k++) {
    cs[k] = cos(2.0 * M_PI * k / padded);
    sn[k] = sin(2.0 * M_PI * k / padded);
  }
  std::vector<double> re(n), im(n);
  for (int k = 0; k < nb; k++) {
    for (int i = 0; i < n; i++) re[i] = im[i] = 0.0;
    for (int j = 0; j < n; j++) {
      const int ph = (int)(((long long)k * j) % padded);
      const double c = cs[ph], s = -sn[ph];
      const double* mj = &m[(size_t)j * n];
      for (int i = 0; i < n; i++) {
        re[i] += c * mj[i];
        im[i] += s * mj[i];
      }
    }
    for (int i = 0; i < n; i++) {
      op[(size_t)k * n + i] = (float)re[i];
      op[(size_t)(nb + k) * n + i] = (float)im[i];
    }
  }
}

// kaldi get_mel_banks without VTLN (oracle/fbank_linear.py: mel_banks): [80][257] float32 + the non-zero range of every filter
void fbank_mel_banks(std::vector<float>& banks, std::vector<int>& k_lo, std::vector<int>& k_hi) {
  const int num_bins = 80, padded = 512, nfft = padded / 2;
  const double sf = 16000.0, low = 20.0, high = 0.5 * sf;
  auto mel = [](double f) { return 1127.0 * log(1.0 + f / 700.0); };
  const double mlow = mel(low), mhigh = mel(high), delta = (mhigh - mlow) / (num_bins + 1), bw = sf / padded;
  banks.assign((size_t)num_bins * 257, 0.f);
  k_lo.assign(num_bins, 0);
  k_hi.assign(num_bins, 0);
  for (int b = 0; b < num_bins; b++) {
    const double left = mlow + b * delta, center = mlow + (b + 1.0) * delta, right = mlow + (b + 2.0) * delta;
    int lo = 257, hi = 0;
    for (int k = 0; k < nfft; k++) {
      const double m = mel(bw * k);
      const double up = (m - left) / (center - left), down = (right - m) / (right - center);
      const double v = fmax(0.0, fmin(up, down));
      banks[(size_t)b * 257 + k] = (float)v;
      if (v > 0.0) {
        lo = k < lo ? k : lo;
        hi = k + 1 > hi ? k + 1 : hi;
      }
    }
    k_lo[b] = lo < hi ? lo : 0;
    k_hi[b] = lo < hi ? hi : 0;
  }
}

}  // namespace dg

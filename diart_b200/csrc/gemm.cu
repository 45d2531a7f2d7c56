// Shifted-window GEMM in float32 on the CUDA cores: the reference that dg_selftest_gemm_tc (tests/test_gpu_gemm_tc.py)
// compares the wgmma split-precision GEMM of gemm_tc.cu against.  No network layer runs on it.
//     C[m, n] = epi( sum_{j<KW} sum_{c<Cin} A[m + j*dil, c] * W[j*Cin + c, n] + bias[n] )
// over a time-major activation matrix (dg_common.cuh, Geom); `epi` is bias, or bias -> LeakyReLU -> BatchNorm1d(eval)
// affine, the two element-wise epilogues of the TDNN layers and the Linear layers.
#include "dg_common.cuh"

namespace dg {

constexpr int BM_T = 128, BN_T = 64, BK_T = 16, G_THREADS = 128;

template <int EPI>
__global__ void __launch_bounds__(G_THREADS) gemm_kernel(GemmArgs a) {
  constexpr int TM = 8;   // rows per thread
  __shared__ __align__(16) float As[2][BK_T][BM_T + 4];
  __shared__ __align__(16) float Ws[2][BK_T][BN_T];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * BM_T;
  const int n0 = blockIdx.y * BN_T;
  const int Ktot = a.KW * a.Cin;
  const int nkb = (Ktot + BK_T - 1) / BK_T;
  const int ty = tid >> 3, tx = tid & 7;   // 16 x 8 threads; thread tile TM x 8

  // ---- A loader: BM rows x 4 float4 per k-block -> BM*4/128 float4 per thread
  constexpr int A_PER = BM_T * 4 / G_THREADS;
  // ---- W loader: 16 rows x 16 float4 -> 2 per thread
  float4 a_reg[A_PER], w_reg[2];

  auto load_tiles = [&](int kb) {
    const int k0 = kb * BK_T;
#pragma unroll
    for (int i = 0; i < A_PER; i++) {
      const int idx = tid + i * G_THREADS;
      const int r = idx >> 2, q = idx & 3;
      const int k = k0 + q * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < Ktot) {
        const int j = k / a.Cin, c = k - j * a.Cin;
        const long long row = m0 + r + (long long)j * a.dil;
        if (row < a.Mtot) v = *reinterpret_cast<const float4*>(a.A + row * a.lda + c);
      }
      a_reg[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int idx = tid + i * G_THREADS;
      const int r = idx >> 4, q = idx & 15;
      const int k = k0 + r, n = n0 + q * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k < Ktot && n < a.ldw) v = *reinterpret_cast<const float4*>(a.W + (size_t)k * a.ldw + n);
      w_reg[i] = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; i++) {
      const int idx = tid + i * G_THREADS;
      const int r = idx >> 2, q = idx & 3;
      As[buf][q * 4 + 0][r] = a_reg[i].x;
      As[buf][q * 4 + 1][r] = a_reg[i].y;
      As[buf][q * 4 + 2][r] = a_reg[i].z;
      As[buf][q * 4 + 3][r] = a_reg[i].w;
    }
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int idx = tid + i * G_THREADS;
      const int r = idx >> 4, q = idx & 15;
      *reinterpret_cast<float4*>(&Ws[buf][r][q * 4]) = w_reg[i];
    }
  };

  float acc[TM][8];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) acc[i][j] = 0.f;

  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kb = 0; kb < nkb; kb++) {
    const int buf = kb & 1;
    if (kb + 1 < nkb) load_tiles(kb + 1);
#pragma unroll
    for (int kk = 0; kk < BK_T; kk++) {
      float av[TM], wv[8];
      const float4 x0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8]);
      const float4 x1 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8 + 4]);
      av[0] = x0.x; av[1] = x0.y; av[2] = x0.z; av[3] = x0.w;
      av[4] = x1.x; av[5] = x1.y; av[6] = x1.z; av[7] = x1.w;
      const float4 w0 = *reinterpret_cast<const float4*>(&Ws[buf][kk][tx * 4]);
      const float4 w1 = *reinterpret_cast<const float4*>(&Ws[buf][kk][32 + tx * 4]);
      wv[0] = w0.x; wv[1] = w0.y; wv[2] = w0.z; wv[3] = w0.w;
      wv[4] = w1.x; wv[5] = w1.y; wv[6] = w1.z; wv[7] = w1.w;
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    if (kb + 1 < nkb) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue.  Thread columns: n0 + tx*4 + {0..3} and n0 + 32 + tx*4 + {0..3}
#pragma unroll
  for (int half = 0; half < 2; half++) {
    const int n = n0 + half * 32 + tx * 4;
    if (n >= a.N) continue;   // N is a multiple of 4 (checked by the launcher)
    float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.bias) bias = *reinterpret_cast<const float4*>(a.bias + n);
    float4 bsc = make_float4(1.f, 1.f, 1.f, 1.f), bsh = make_float4(0.f, 0.f, 0.f, 0.f);
    if (EPI == EPI_BIAS_LEAKY_BN) {
      bsc = *reinterpret_cast<const float4*>(a.bn_scale + n);
      bsh = *reinterpret_cast<const float4*>(a.bn_shift + n);
    }
#pragma unroll
    for (int i = 0; i < TM; i++) {
      const long long m = m0 + ty * TM + i;
      if (m >= a.M) continue;
      float4 v = make_float4(acc[i][half * 4 + 0] + bias.x, acc[i][half * 4 + 1] + bias.y,
                             acc[i][half * 4 + 2] + bias.z, acc[i][half * 4 + 3] + bias.w);
      if (EPI == EPI_BIAS_LEAKY_BN) {
        v.x = leaky(v.x); v.y = leaky(v.y); v.z = leaky(v.z); v.w = leaky(v.w);
        v.x = fmaf(v.x, bsc.x, bsh.x); v.y = fmaf(v.y, bsc.y, bsh.y);
        v.z = fmaf(v.z, bsc.z, bsh.z); v.w = fmaf(v.w, bsc.w, bsh.w);
      }
      *reinterpret_cast<float4*>(a.C + m * a.ldc + n) = v;
    }
  }
}

int launch_gemm(const GemmArgs& a, cudaStream_t st) {
  ProfScope _ps(a.tag ? a.tag : "gemm", st);
  if (a.Cin % 4 || a.lda % 4 || a.ldw % 4 || a.ldc % 4 || a.N % 4) {
    set_error("gemm: channel counts must be multiples of 4");
    return -1;
  }
  const dim3 grid((unsigned)((a.M + BM_T - 1) / BM_T), (a.N + BN_T - 1) / BN_T);
  if (a.epi == EPI_BIAS) gemm_kernel<EPI_BIAS><<<grid, G_THREADS, 0, st>>>(a);
  else gemm_kernel<EPI_BIAS_LEAKY_BN><<<grid, G_THREADS, 0, st>>>(a);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

// Bidirectional LSTM recurrence of PyanNet on the tensor cores (wgmma), split precision (hi + lo fp16 planes).
// (nn.LSTM(60,128,num_layers=4,bidirectional), SURVEY.md Appendix A.3; reached from the reference through
// src/diart/models.py:131-133.)  The input projections are hoisted into gemm_tc.cu; this kernel runs the 293
// dependent steps of one layer.
//
// One CTA owns 8 batch rows of one direction and ALL 4 x 128 gate rows, so a step is
//     gates[512, 8] = W_hh[512, 128] . h_{t-1}^T[128, 8]          (M = gate rows, N = batch rows)
// computed by four warpgroups, 128 gate rows (two m64 tiles) each.  The gate rows are PERMUTED when the weights are packed
// (lstm_tc_pack_whh) so that the accumulator fragment of a thread holds i, f (tile 0) and g, o (tile 1) of one hidden unit
// for two batch rows: the thread updates c and h of those cells with no cross-thread exchange.
//
//  * W_hh stays on the SM for the whole sequence: the hi plane in REGISTERS (the A operand of wgmma may come from registers:
//    64 per thread), the lo plane in shared memory (128 KB, 128B-swizzled, one TMA load).  Products per k-step:
//    Whi.hlo and Whi.hhi (A from registers), Wlo.hhi (A from shared memory).
//  * h_t is the B operand, K-major without swizzle: unit-contiguous 16-byte units of 8 hidden units per batch row, double
//    buffered; one CTA barrier per step hands it to the next step's MMAs.
//  * The cell update needs 7 MUFU operations (one reciprocal for f*c + i*g, one for o*tanh(c)); rows past the batch are
//    skipped.
//  * h_t leaves the kernel as the hi/lo planes the next layer's GEMM reads (no float32 round trip, no split kernel).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "dg_common.cuh"
#include "tc_ptx.cuh"

namespace dg {

constexpr int LT_NB = 8;                                // batch rows per CTA (N of every MMA)
constexpr int LT_THREADS = 512;                         // four warpgroups
constexpr int LT_WS_BYTES = 2 * 512 * 128;              // W_lo of one direction: 2 k-blocks x (512 rows x 128 B)
constexpr int LT_PLANE = 128 * LT_NB * 2;               // one plane of h_t: 16 unit groups x 8 rows x 16 B = 2 KB
constexpr int LT_H_BYTES = 2 * 2 * LT_PLANE;            // [buffer][plane]
constexpr int LT_SMEM = LT_WS_BYTES + LT_H_BYTES + 64 + 1024;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// packed gate row of (unit u, gate g): warpgroup u / 32 owns units 32 wg .. 32 wg + 31; in its tile t = g / 2, warp w = (u % 32) / 8
// owns rows 16 w .. 16 w + 15: row 16 w + u % 8 holds gate 2 t, row 16 w + 8 + u % 8 gate 2 t + 1
__host__ __device__ constexpr int lt_row(int g, int u) { return (u >> 5) * 128 + (g >> 1) * 64 + ((u & 31) >> 3) * 16 + (g & 1) * 8 + (u & 7); }

__global__ void __launch_bounds__(LT_THREADS, 1)
lstm_tc_kernel(const __grid_constant__ CUtensorMap tm_wlo, const float* __restrict__ gx /*[item][frame][1024]*/,
               const uint16_t* __restrict__ w_hi /*[2][512][128], packed rows*/, int B, int T, int stride, int groups_per_dir,
               float* __restrict__ hout, uint16_t* __restrict__ out_hi, uint16_t* __restrict__ out_lo, float acc_scale) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* wsm = smem;                         // [k-block][512 x 128 B]   (W_lo)
  unsigned char* hsm = smem + LT_WS_BYTES;           // [buffer][plane][2 KB]
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + LT_WS_BYTES + LT_H_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wq = warp & 3;
  const int dir = blockIdx.x / groups_per_dir;
  const int b0 = (blockIdx.x - dir * groups_per_dir) * LT_NB;

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < LT_H_BYTES / 4; i += LT_THREADS) reinterpret_cast<uint32_t*>(hsm)[i] = 0u;   // h_0 = 0
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(w_full, LT_WS_BYTES);
    for (int kb = 0; kb < 2; kb++)
      for (int half = 0; half < 2; half++)
        tma_load_2d(wsm + kb * 65536 + half * 32768, &tm_wlo, kb * 64, dir * 512 + half * 256, w_full);
  }
  // W_hi as A fragments: tile t, k-step ks -> rows r0 = 16 wq + lane / 4 and r0 + 8 of the tile, k = 16 ks + 2 (lane % 4) (+ 8)
  uint32_t wa[2][8][4];
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(w_hi + (size_t)dir * 512 * 128);
#pragma unroll
    for (int t = 0; t < 2; t++) {
      const int r0 = wg * 128 + t * 64 + wq * 16 + (lane >> 2);
#pragma unroll
      for (int ks = 0; ks < 8; ks++) {
        const int k2 = (ks * 16 + 2 * (lane & 3)) >> 1;     // in 32-bit pairs
        wa[t][ks][0] = src[(size_t)r0 * 64 + k2];
        wa[t][ks][1] = src[(size_t)(r0 + 8) * 64 + k2];
        wa[t][ks][2] = src[(size_t)r0 * 64 + k2 + 4];
        wa[t][ks][3] = src[(size_t)(r0 + 8) * 64 + k2 + 4];
      }
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // zeroed h buffers -> visible to the tensor core
  __syncthreads();
  mbar_wait(w_full, 0);

  const int u = wg * 32 + wq * 8 + (lane >> 2);      // hidden unit of this thread
  const int n0 = 2 * (lane & 3);                      // its two batch columns n0, n0 + 1
  bool valid[2];
  for (int e = 0; e < 2; e++) valid[e] = b0 + n0 + e < B;
  const int t0 = dir == 0 ? 0 : T - 1;
  const ptrdiff_t dh = dir == 0 ? 256 : -256;
  const size_t row_h = (size_t)stride * 256;
  const size_t e0 = ((size_t)(b0 + n0) * stride + t0) * 256 + dir * 128 + u;
  float* hp = hout ? hout + e0 : nullptr;
  uint16_t* php = out_hi ? out_hi + e0 : nullptr;
  const size_t plane_off = out_hi ? (size_t)(out_lo - out_hi) : 0;
  const float* xp = gx + ((size_t)(b0 + n0) * stride + t0) * 1024 + dir * 512 + u;
  const ptrdiff_t dx = dir == 0 ? 1024 : -1024;
  const size_t row_x = (size_t)stride * 1024;
  // shared address of (unit u, batch row n0) in buffer 0, hi plane; row n0 + 1 is 16 bytes further
  const uint32_t h_addr = smem_u32(hsm) + (u >> 3) * 128 + n0 * 16 + (u & 7) * 2;
  const uint32_t wlo = smem_u32(wsm) + (wg * 128) * 128;
  const float L2E = 1.4426950408889634f;
  float c[2] = {0.f, 0.f};
  for (int step = 0; step < T; step++) {
    const int buf = step & 1;
    const uint32_t hb = smem_u32(hsm) + buf * (LT_H_BYTES / 2);
    float acc[2][4];
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ks++) {
      // B = h_{t-1}: K-major, 8 units x 8 rows per 128-byte core matrix, k-step = two core matrices
      const uint64_t bh = wg_desc_plain(hb + ks * 256, 128, 128), bl = wg_desc_plain(hb + LT_PLANE + ks * 256, 128, 128);
#pragma unroll
      for (int t = 0; t < 2; t++) {
        const uint64_t al = wg_desc(wlo + (ks >> 2) * 65536 + t * 64 * 128) + (uint64_t)(((ks & 3) * 32) >> 4);
        wgmma_rs<8>(acc[t], wa[t][ks], bl, ks != 0);      // W_hi . h_lo
        wgmma_ss<8>(acc[t], al, bh, 1);                   // W_lo . h_hi
        wgmma_rs<8>(acc[t], wa[t][ks], bh, 1);            // W_hi . h_hi
      }
    }
    wg_commit();
    // the gate pre-activations of this step, under the MMAs
    float xg[4][2];
#pragma unroll
    for (int g = 0; g < 4; g++)
#pragma unroll
      for (int e = 0; e < 2; e++) xg[g][e] = valid[e] ? __ldg(xp + e * row_x + g * 128) : 0.f;
    xp += dx;
    wg_wait<0>();
    wg_fence_acc(acc[0]);
    wg_fence_acc(acc[1]);
    float h[2];
    uint16_t hh[2], hl[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
      // exponents capped at 2^40: sigmoid floor 9e-13, products stay below 2^127
      const float di = 1.f + ex2_approx(fminf(fmaf(acc[0][e], acc_scale, xg[0][e]) * -L2E, 40.f));       // 1 + e^-i
      const float df = 1.f + ex2_approx(fminf(fmaf(acc[0][2 + e], acc_scale, xg[1][e]) * -L2E, 40.f));   // 1 + e^-f
      const float eg = ex2_approx(fminf(fmaf(acc[1][e], acc_scale, xg[2][e]) * (2.f * L2E), 40.f));
      // c' = c / (1 + ef) + (eg - 1) / ((1 + ei)(1 + eg))  over one common denominator
      const float p = di * (1.f + eg);
      c[e] = fmaf(c[e], p, (eg - 1.f) * df) * rcp_approx(p * df);
      const float ec = ex2_approx(fminf(c[e] * (2.f * L2E), 40.f));
      // h = tanh(c') / (1 + e^-o)
      const float eo = ex2_approx(fminf(fmaf(acc[1][2 + e], acc_scale, xg[3][e]) * -L2E, 40.f));
      h[e] = valid[e] ? (ec - 1.f) * rcp_approx((1.f + eo) * (ec + 1.f)) : 0.f;
      split_h16(h[e], hh[e], hl[e]);
    }
    const uint32_t dst = h_addr + (buf ^ 1) * (LT_H_BYTES / 2);
#pragma unroll
    for (int e = 0; e < 2; e++) {
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(dst + e * 16), "h"(hh[e]) : "memory");
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(dst + LT_PLANE + e * 16), "h"(hl[e]) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // the copies of h_t for the next layer leave after the hand-off: they are not on the recurrence's critical path
#pragma unroll
    for (int e = 0; e < 2; e++)
      if (valid[e]) {
        if (php) {      // the next layer's GEMM reads h as hi/lo planes: written directly (no float32 round trip)
          php[e * row_h] = hh[e];
          php[e * row_h + plane_off] = hl[e];
        }
        if (hp) hp[e * row_h] = h[e];
      }
    if (php) php += dh;
    if (hp) hp += dh;
  }
}

size_t lstm_tc_plane_elems() { return (size_t)2 * 512 * 128; }

// torch weight_hh_l{L}[_reverse] ([512][128], gate order i,f,g,o) -> fp16 hi / lo planes [2][512][128], rows in the kernel's
// order (lt_row); returns the power-of-two factor both planes were multiplied by (weight_plane_scale; one factor for both
// directions)
float lstm_tc_pack_whh(const float* whh_fwd, const float* whh_bwd, uint16_t* hi, uint16_t* lo) {
  const float s0 = weight_plane_scale(whh_fwd, 512 * 128), s1 = weight_plane_scale(whh_bwd, 512 * 128);
  const float scale = s0 < s1 ? s0 : s1;
  std::vector<float> perm((size_t)512 * 128);
  for (int d = 0; d < 2; d++) {
    const float* w = d == 0 ? whh_fwd : whh_bwd;
    for (int g = 0; g < 4; g++)
      for (int u = 0; u < 128; u++) memcpy(&perm[(size_t)lt_row(g, u) * 128], w + ((size_t)g * 128 + u) * 128, 128 * sizeof(float));
    split_weights_host(perm.data(), 512, 512, 128, hi + (size_t)d * 512 * 128, lo + (size_t)d * 512 * 128, scale);
  }
  return scale;
}

int launch_lstm_layer_tc(const float* gx, const void* whh_hi, const void* whh_lo, float w_scale, int B, int T, int stride,
                         float* hout, void* out_hi, void* out_lo, cudaStream_t st) {
  ProfScope _ps("lstm_rec", st);
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return -2;
  }
  if (!hout && !out_hi) {
    set_error("lstm_rec: no output buffer");
    return -1;
  }
  CUtensorMap tm;
  cuuint64_t dims[2] = {128, 1024};
  cuuint64_t strides[1] = {256};
  cuuint32_t box[2] = {64, 256};
  cuuint32_t estr[2] = {1, 1};
  // shared-memory-resident plane = lo, register-resident plane = hi (see the MMA sequence in the kernel)
  if (fn(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(whh_lo), dims, strides, box, estr,
         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed for W_hh");
    return -2;
  }
  auto kern = lstm_tc_kernel;
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done)) DG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, LT_SMEM));
  const int gpd = (B + LT_NB - 1) / LT_NB;
  const float inv = w_scale > 0.f ? 1.f / w_scale : 1.f;
  kern<<<2 * gpd, LT_THREADS, LT_SMEM, st>>>(tm, gx, reinterpret_cast<const uint16_t*>(whh_hi), B, T, stride, gpd, hout,
                                             reinterpret_cast<uint16_t*>(out_hi), reinterpret_cast<uint16_t*>(out_lo), inv);
  DG_LAUNCHED();
  return 0;
}

int lstm_tc_ctas(int B) { return 2 * ((B + LT_NB - 1) / LT_NB); }

}  // namespace dg

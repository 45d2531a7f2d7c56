// Bidirectional LSTM recurrence of PyanNet on the tensor cores (wgmma), split precision (hi + lo fp16 planes).
// (nn.LSTM(60,128,num_layers=4,bidirectional), SURVEY.md Appendix A.3; reached from the reference through
// src/diart/models.py:131-133.)  The input projections are hoisted into gemm_tc.cu; this kernel runs the 293
// dependent steps of one layer.
//
// One CTA owns 16 batch rows of one direction and ALL 4 x 128 gate rows, so a step is
//     gates[512, 16] = W_hh[512, 128] . h_{t-1}^T[128, 16]        (M = gate rows, N = batch rows)
// computed by four warpgroups, 128 gate rows (two m64 tiles) each.  The gate rows are PERMUTED when the weights are packed
// (lstm_tc_pack_whh) so that the accumulator fragment of a thread holds i, f (tile 0) and g, o (tile 1) of one hidden unit
// for four batch rows (n0, n0 + 1, n0 + 8, n0 + 9): the thread updates c and h of those cells with no cross-thread
// exchange.  16 rows per CTA keep the recurrence on 2 x ceil(B / 16) SMs; the rest run the other streams' GEMMs.
// An 8-row instance (m64n8, two cells per thread) serves small batches (lt_rows).
//
//  * W_hh stays on the SM for the whole sequence: the hi plane in REGISTERS (the A operand of wgmma may come from registers:
//    64 per thread), the lo plane in shared memory (128 KB, 128B-swizzled, one TMA load).  Products per k-step:
//    Whi.hlo and Whi.hhi (A from registers), Wlo.hhi (A from shared memory).
//  * h_t is the B operand, K-major without swizzle: unit-contiguous 16-byte units of 8 hidden units per batch row, two
//    8-row core matrices along N, double buffered; one CTA barrier per step hands it to the next step's MMAs.
//  * The gate pre-activations of a step (512 float32 columns x 16 rows) arrive by TMA in a two-slot ring: one thread loads
//    step t + 1 into the other slot while step t's MMAs run, and the step's CTA barrier tells it the slot has been read.
//    The box is 128B-swizzled (32 columns x NB rows per group), so a warp's reads of one gate (8 units x 4 rows) hit 32
//    different banks.  Rows past the batch are zero-filled by TMA: nothing past the buffer is read.
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

constexpr int LT_THREADS = 512;                         // four warpgroups
constexpr int LT_WS_BYTES = 2 * 512 * 128;              // W_lo of one direction: 2 k-blocks x (512 rows x 128 B)
// per instance of NB batch rows per CTA (N of every MMA)
__host__ __device__ constexpr int lt_plane(int nb) { return 128 * nb * 2; }                 // one plane of h_t: 16 unit groups x nb rows x 16 B
__host__ __device__ constexpr int lt_h_bytes(int nb) { return 2 * 2 * lt_plane(nb); }       // [buffer][plane]
__host__ __device__ constexpr int lt_x_bytes(int nb) { return 512 * nb * 4; }               // one ring slot: a step's gate pre-activations
constexpr int lt_smem(int nb) { return LT_WS_BYTES + lt_h_bytes(nb) + 2 * lt_x_bytes(nb) + 64 + 1024; }
static_assert(lt_smem(16) <= 227 * 1024, "lstm_tc: shared memory over the per-block limit");
// 16 rows per CTA from 128 windows up: there the SMs the recurrence frees run the concurrent GEMMs of the pipelined step.
// Smaller batches (the sub-batches of a synchronous call) wait for the recurrence itself, whose step is shorter at 8 rows.
// Each output element takes the same products in the same order in both instances: rows are bit-identical.
static int lt_rows(int B) { return B >= 128 ? 16 : 8; }

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

template <int NB>
__global__ void __launch_bounds__(LT_THREADS, 1)
lstm_tc_kernel(const __grid_constant__ CUtensorMap tm_wlo, const __grid_constant__ CUtensorMap tm_gx,
               const uint16_t* __restrict__ w_hi /*[2][512][128], packed rows*/, int B, int T, int stride, int groups_per_dir,
               float* __restrict__ hout, uint16_t* __restrict__ out_hi, uint16_t* __restrict__ out_lo, float acc_scale) {
  constexpr int LT_PLANE = lt_plane(NB), LT_H_BYTES = lt_h_bytes(NB), LT_X_BYTES = lt_x_bytes(NB);
  constexpr int E = NB / 4;                          // cells per thread
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* wsm = smem;                         // [k-block][512 x 128 B]   (W_lo)
  unsigned char* hsm = smem + LT_WS_BYTES;           // [buffer][plane]
  unsigned char* xsm = hsm + LT_H_BYTES;             // [slot][16 column groups][NB rows][32 columns], 128B-swizzled
  uint64_t* w_full = reinterpret_cast<uint64_t*>(xsm + 2 * LT_X_BYTES);
  uint64_t* x_full = w_full + 1;                     // [slot]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wq = warp & 3;
  const int dir = blockIdx.x / groups_per_dir;
  const int b0 = (blockIdx.x - dir * groups_per_dir) * NB;
  const int t0 = dir == 0 ? 0 : T - 1;
  const int dt = dir == 0 ? 1 : -1;

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    mbar_init(&x_full[0], 1);
    mbar_init(&x_full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < LT_H_BYTES / 4; i += LT_THREADS) reinterpret_cast<uint32_t*>(hsm)[i] = 0u;   // h_0 = 0
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(w_full, LT_WS_BYTES);
    for (int kb = 0; kb < 2; kb++)
      for (int half = 0; half < 2; half++)
        tma_load_2d(wsm + kb * 65536 + half * 32768, &tm_wlo, kb * 64, dir * 512 + half * 256, w_full);
    // gate map coordinates: {column in group, item, column group, frame}
    mbar_expect_tx(&x_full[0], LT_X_BYTES);
    tma_load_4d(xsm, &tm_gx, 0, b0, dir * 16, t0, &x_full[0]);
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
  const int n0 = 2 * (lane & 3);                      // its batch rows n0 + ne(e), e < E
  auto ne = [](int e) { return (e & 1) + 8 * (e >> 1); };
  bool valid[E];
#pragma unroll
  for (int e = 0; e < E; e++) valid[e] = b0 + n0 + ne(e) < B;
  // output row (item b0 + n0, this step's frame); the addresses are formed at the stores, so that no 64-bit pointer stays
  // live across the MMAs (with per-row pointers ptxas spills at the 128-register budget)
  int hrow = (b0 + n0) * stride + t0;
  // shared address of gate 0 (i) of unit u for batch rows n0 and n0 + 1 in slot 0: column group wg, 128-byte row n0 (+ 1),
  // 16-byte chunk (u % 32) / 4 xor the row's low three bits; gate g is 4 groups further, rows n0 + 8 and n0 + 9 1 KB
  uint32_t x_addr[2];
#pragma unroll
  for (int j = 0; j < 2; j++) x_addr[j] = smem_u32(xsm) + wg * NB * 128 + (n0 + j) * 128 + ((((u & 31) >> 2) ^ (n0 + j)) << 4) + (u & 3) * 4;
  // shared address of (unit u, batch row n0) in buffer 0, hi plane; row n0 + 1 is 16 bytes further, rows n0 + 8 and
  // n0 + 9 one core matrix (128 bytes)
  const uint32_t h_addr = smem_u32(hsm) + (u >> 3) * NB * 16 + n0 * 16 + (u & 7) * 2;
  const uint32_t wlo0 = smem_u32(wsm) + (wg * 128) * 128;
  const float L2E = 1.4426950408889634f;
  float c[E] = {};
  for (int step = 0; step < T; step++) {
    const int buf = step & 1;
    const uint32_t hb = smem_u32(hsm) + buf * (LT_H_BYTES / 2);
    // opaque per step: ptxas would otherwise hoist the 16 W_lo descriptors and the gate addresses out of the loop and spill
    uint32_t wlo = wlo0;
    asm volatile("" : "+r"(wlo));
    float acc[2][NB / 2];
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ks++) {
      // B = h_{t-1}: K-major, 8 units x 8 rows per 128-byte core matrix; a k-step is two core matrices along K (NB x 16
      // bytes apart) by NB / 8 along N (128 bytes apart)
      const uint64_t bh = wg_desc_plain(hb + ks * NB * 32, NB * 16, 128),
                     bl = wg_desc_plain(hb + LT_PLANE + ks * NB * 32, NB * 16, 128);
#pragma unroll
      for (int t = 0; t < 2; t++) {
        const uint64_t al = wg_desc(wlo + (ks >> 2) * 65536 + t * 64 * 128) + (uint64_t)(((ks & 3) * 32) >> 4);
        wgmma_rs<NB>(acc[t], wa[t][ks], bl, ks != 0);     // W_hi . h_lo
        wgmma_ss<NB>(acc[t], al, bh, 1);                  // W_lo . h_hi
        wgmma_rs<NB>(acc[t], wa[t][ks], bh, 1);           // W_hi . h_hi
      }
    }
    wg_commit();
    // the next step's gate pre-activations, under the MMAs: its slot was last read in step - 1, before that step's barrier
    if (threadIdx.x == 0 && step + 1 < T) {
      uint64_t* bar = &x_full[(step + 1) & 1];
      mbar_expect_tx(bar, LT_X_BYTES);
      tma_load_4d(xsm + ((step + 1) & 1) * LT_X_BYTES, &tm_gx, 0, b0, dir * 16, t0 + (step + 1) * dt, bar);
    }
    wg_wait<0>();
    wg_fence_acc(acc[0]);
    wg_fence_acc(acc[1]);
    mbar_wait(&x_full[buf], (step >> 1) & 1);
    float h[E];
    uint16_t hh[E], hl[E];
#pragma unroll
    for (int e = 0; e < E; e++) {
      // accumulator of row n0 + ne(e): gates i, g at index 4 (e / 2) + e % 2, gates f, o two further
      const int a = 4 * (e >> 1) + (e & 1);
      const uint32_t xa = x_addr[e & 1] + buf * LT_X_BYTES + (e >> 1) * 1024;
      float xg[4];
#pragma unroll
      for (int g = 0; g < 4; g++) asm volatile("ld.shared.f32 %0, [%1];" : "=f"(xg[g]) : "r"(xa + g * 4 * NB * 128) : "memory");
      // exponents capped at 2^40: sigmoid floor 9e-13, products stay below 2^127
      const float di = 1.f + ex2_approx(fminf(fmaf(acc[0][a], acc_scale, xg[0]) * -L2E, 40.f));       // 1 + e^-i
      const float df = 1.f + ex2_approx(fminf(fmaf(acc[0][a + 2], acc_scale, xg[1]) * -L2E, 40.f));   // 1 + e^-f
      const float eg = ex2_approx(fminf(fmaf(acc[1][a], acc_scale, xg[2]) * (2.f * L2E), 40.f));
      // c' = c / (1 + ef) + (eg - 1) / ((1 + ei)(1 + eg))  over one common denominator
      const float p = di * (1.f + eg);
      c[e] = fmaf(c[e], p, (eg - 1.f) * df) * rcp_approx(p * df);
      const float ec = ex2_approx(fminf(c[e] * (2.f * L2E), 40.f));
      // h = tanh(c') / (1 + e^-o)
      const float eo = ex2_approx(fminf(fmaf(acc[1][a + 2], acc_scale, xg[3]) * -L2E, 40.f));
      h[e] = valid[e] ? (ec - 1.f) * rcp_approx((1.f + eo) * (ec + 1.f)) : 0.f;
      split_h16(h[e], hh[e], hl[e]);
    }
    const uint32_t dst = h_addr + (buf ^ 1) * (LT_H_BYTES / 2);
#pragma unroll
    for (int e = 0; e < E; e++) {
      const uint32_t o = (e & 1) * 16 + (e >> 1) * 128;
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(dst + o), "h"(hh[e]) : "memory");
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(dst + LT_PLANE + o), "h"(hl[e]) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // the copies of h_t for the next layer leave after the hand-off: they are not on the recurrence's critical path
#pragma unroll
    for (int e = 0; e < E; e++)
      if (valid[e]) {
        const size_t o = (size_t)(hrow + ne(e) * stride) * 256 + dir * 128 + u;
        if (out_hi) {      // the next layer's GEMM reads h as hi/lo planes: written directly (no float32 round trip)
          out_hi[o] = hh[e];
          out_lo[o] = hl[e];
        }
        if (hout) hout[o] = h[e];
      }
    hrow += dt;
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
  // gate pre-activations [item][frame][1024] as {32 columns, item, column group, frame}: one box is a step's 512 columns of
  // one direction for the CTA's items, stored [group][item][32 columns] so that the 128B swizzle spreads a warp's rows over the
  // banks.  The item extent is exactly B: rows of a partial last CTA are zero-filled, not read past the batch.
  const int nb = lt_rows(B);
  CUtensorMap tmx;
  cuuint64_t xdims[4] = {32, (cuuint64_t)B, 32, (cuuint64_t)T};
  cuuint64_t xstrides[3] = {(cuuint64_t)stride * 4096, 128, 4096};
  cuuint32_t xbox[4] = {32, (cuuint32_t)nb, 16, 1};
  cuuint32_t xestr[4] = {1, 1, 1, 1};
  if (fn(&tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(gx), xdims, xstrides, xbox, xestr,
         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed for the LSTM gate rows");
    return -2;
  }
  auto kern = nb == 16 ? lstm_tc_kernel<16> : lstm_tc_kernel<8>;
  const int smem = lt_smem(nb);
  static bool attr_done[2][64] = {};
  if (first_use_on_device(attr_done[nb == 16])) DG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int gpd = (B + nb - 1) / nb;
  const float inv = w_scale > 0.f ? 1.f / w_scale : 1.f;
  kern<<<2 * gpd, LT_THREADS, smem, st>>>(tm, tmx, reinterpret_cast<const uint16_t*>(whh_hi), B, T, stride, gpd, hout,
                                          reinterpret_cast<uint16_t*>(out_hi), reinterpret_cast<uint16_t*>(out_lo), inv);
  DG_LAUNCHED();
  return 0;
}

int lstm_tc_rows(int B) { return lt_rows(B); }
int lstm_tc_ctas(int B) { return 2 * ((B + lt_rows(B) - 1) / lt_rows(B)); }

}  // namespace dg

// Shifted-window GEMM on the Hopper tensor cores (wgmma + TMA), hi/lo split precision.
//
//     C[m, n] = epi( sum_{j<KW} sum_{c<Cin} A[m + j*dil, c] * W[n, j*Cin + c] + bias[n] )
//
// The dense contractions of the path -- the five TDNN layers of XVectorSincNet (dilated Conv1d ->
// LeakyReLU -> BatchNorm1d(eval)) and the LSTM input projections of PyanNet (SURVEY.md Appendix
// A.3/A.4; reached from the reference through src/diart/models.py:131-133) -- must stay at float32-level
// accuracy because their outputs feed hard thresholds (tau_active, rho_update, delta_new).  Each float32
// operand x is therefore carried as two fp16 planes, hi = rn16(x) and lo = rn16(x - hi) (22 significand bits
// for the pair), and every k-step issues three wgmma (hi*hi + lo*hi + hi*lo) into the same float32 register
// accumulator.  Measured against the float32 reference GEMM of gemm.cu: < 1e-5 relative (tests/test_gpu_gemm_tc.py).
//
// Because activations are stored time-major ([item][row][channel]) a Conv1d tap is just a TMA box whose
// row coordinate is shifted by j*dil: no im2col is ever materialised.
//
// One kernel, gemm_tc_kernel, for every epilogue.  CTA = 384 threads, persistent over 128 x BN tiles:
//   warpgroup 0     (setmaxnreg 40) one thread hands the CTA's tiles to the two consumers alternately and loads per k-block
//                   four boxes (A_hi, A_lo: 128 rows x 32 ch; W_hi, W_lo: BN rows x 32 ch) into a 64B-swizzled ring,
//                   completion on full[] mbarriers
//   warpgroups 1-2  (setmaxnreg 232) ping-pong consumers: each runs whole tiles, 12 wgmma per k-block (two m64 halves x
//                   two k-steps x three products) into registers, a slot is released one k-block later; an ordering
//                   barrier hands the tensor cores to the other consumer once a tile's MMAs are issued, so one consumer's
//                   epilogue overlaps the other's mainloop.
// Tile order: the element-wise epilogues (bias, LeakyReLU + BatchNorm, Conv2d) take the static order b, b + grid, ...;
// the pooling epilogues (TC_POOL, TC_MAXPOOL3), whose cross-row reductions take about as long as the tile's MMAs, take
// tiles in m-major order from a per-stream atomic counter (a CTA that becomes resident late runs fewer tiles).
// Epilogues:
//   element-wise    the two consumers share ONE full-tile staging buffer.  A consumer waits until the other one's data has
//                   left it (a named-barrier pair), then
//                   - bias, LeakyReLU + BatchNorm -> float32 rows or the next layer's hi/lo 16-bit planes: applies the
//                     epilogue to its accumulator fragments in registers and writes the results into 128B-swizzled boxes
//                     (float32: 32 columns x 128 rows; planes: 64 x 128 per plane), which one thread stores with TMA.  The
//                     hardware clips the boxes at rows M and columns N.  The buffer is handed on once TMA has read it.
//                   - Conv2d: writes its whole accumulator as [128][BN + 4] float32 and runs the epilogue from it (row m of
//                     the tile -> thread m: output-row remapping, residual reads, stride-2 subsampling).
//                   One buffer is enough: a consumer needs it only after its own mainloop, and the other consumer runs its
//                   epilogue during that mainloop.
//   pooling         the accumulator goes to the consumer's own shared memory 64 columns at a time, already through bias /
//                   LeakyReLU / BatchNorm (TC_POOL) or the weight scale (TC_MAXPOOL3).
// Every output element gets the same wgmma sequence (k order, lo.hi, hi.lo, hi.hi per k-step) and the same epilogue
// arithmetic whichever CTA or warpgroup runs its tile, so results do not depend on the grid.
#include <cuda.h>
#include <cuda_bf16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "dg_common.cuh"
#include "host.cuh"
#include "tc_ptx.cuh"

namespace dg {

constexpr int TC_BM = 128, TC_BK = 32, TC_THREADS = 384;
constexpr int TC_SMEM_MAX = 227 * 1024;                 // dynamic shared memory per CTA on sm_90

struct TcArgs {
  long long M;          // output rows
  int N;                // valid output channels
  int m_tiles, n_tiles;
  int KW, dil, cin_blocks;
  const float* bias;
  const float* bn_scale;
  const float* bn_shift;
  float* out_f32;       // EPI_F32*: [M, ldc]
  __nv_bfloat16* out_hi;   // EPI_*_SPLIT: [M, ldc] each
  __nv_bfloat16* out_lo;
  int ldc;
  float acc_scale;      // 1 / (power-of-two scale of the weight planes): applied to the accumulator in the epilogue
  int tap_off[9];       // row offset of every tap (Conv1d: j * dil; Conv2d on a zero-padded map: (dw-1) * Hp + (dh-1))
  // TC_CONV2D: rows are positions (item, w, h) of a zero-padded [Wp][Hp] map; outputs go to the padded map [Wop][Hop] of the
  // next layer (stride 1: same geometry; stride 2: computed at every centre, only odd (w, h) are kept)
  int Wp, Hp, Wop, Hop, stride2, relu;
  const __nv_bfloat16* res_hi;   // residual planes in the output geometry, or null
  const __nv_bfloat16* res_lo;
  // TC_POOL: weighted statistics pooling fused into the epilogue (the activation map is never written)
  const float* pool_w;     // [rows][4]: pooling weight of (row, speaker), zero for rows past an item's valid frames
  float* pool_part;        // [m_tiles][2 (item of the tile)][TC_POOL_SLOTS][N]: 4 (speaker) x 2 (sum w e, sum w e^2), pivot;
                           // e = d - pivot
  int pool_item_rows, pool_K, pool_T;   // pool_T: valid frames of an item (its later rows hold garbage and weight 0)
  // TC_MAXPOOL3: m-tiles advance by `tile_rows` <= 126 rows (whole pooling windows, a divisor of the item's rows, so that every
  // item is summed in the same grouping wherever it sits in the batch; the MMA still covers 128 rows), out_f32 receives
  // bias + MaxPool1d(3) over rows ([M / 3, ldc]), pool_part the per-tile InstanceNorm partial sums of the pre-bias pooled values:
  // [m_tiles][2 (item of the tile)][TC_POOL3_SLOTS][N] = (sum, sum of squares) of v - pivot over the pooled frames < pool3_T of
  // an item, pivot
  int tile_rows, pool3_T;
  unsigned* tile_ctr;      // pooling epilogues, [2]: tiles handed out past the first wave, CTAs finished (both back to 0)
  // halo operand mode (gemm_tc_kernel<.., true>): a tile's A operand is its halo, rows m0 .. m0 + halo_rows - 1 of all cin
  // channels, loaded once per tile as [hi | lo][ceil(cin / 32)] boxes of halo_rows x 32 channels (64B swizzle)
  int halo_rows;           // rows of a halo box (tc_halo_rows)
  int cin;                 // channels per tap, a multiple of 16 (no k16 step straddles a tap)
  int wblocks;             // W k-blocks per tile: ceil(KW * cin / 32), two k16 steps each
  int halo_bytes;          // one consumer's halo slot (a multiple of 1 KB)
  int op_bytes;            // the operand region: tap-box ring, or the two halo slots + the W ring
};

enum TcEpi { TC_BIAS_F32 = 0, TC_LEAKY_BN_SPLIT = 1, TC_LEAKY_BN_F32 = 2, TC_CONV2D = 3, TC_POOL = 4, TC_MAXPOOL3 = 5 };

__host__ __device__ constexpr bool tc_pooling(int epi) { return epi == TC_POOL || epi == TC_MAXPOOL3; }
// epilogues whose output tile leaves as TMA boxes
__host__ __device__ constexpr bool tc_box_store(int epi) { return epi == TC_BIAS_F32 || epi == TC_LEAKY_BN_SPLIT || epi == TC_LEAKY_BN_F32; }

// Layout: [operands] [element-wise: the shared staging tile] [barriers] [consumer 0: parameters | pooling: chunk | pooling
// staging] [consumer 1: the same].  Operands, tap-box mode: NSTAGE stages of (A hi, A lo, W hi, W lo); halo mode: the halo
// slots of consumer 0 and 1, then NSTAGE_HALO stages of (W hi, W lo).  Every operand block is a multiple of 1 KB, so the
// staging tile keeps the 1 KB alignment of 128B-swizzled boxes.
template <int BN>
struct TcSmem {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;     // 8 KB per plane
  static constexpr int W_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * W_BYTES;
  static constexpr int W_STAGE_BYTES = 2 * W_BYTES;
  // 128 / 144 / 120 KB of operands in flight at BN = 128 / 64 / 32
  static constexpr int NSTAGE = BN == 128 ? 4 : 6;
  static constexpr int NSTAGE_HALO = BN == 128 ? 5 : 6;   // 80 / 48 KB of W in flight
  // halo slot of `cin` channels x `rows` rows, hi and lo planes
  __host__ static int halo_bytes(int cin, int rows) { return (2 * ((cin + 31) / 32) * rows * 64 + 1023) / 1024 * 1024; }
  __host__ static int halo_op_bytes(int cin, int rows) { return 2 * halo_bytes(cin, rows) + NSTAGE_HALO * W_STAGE_BYTES; }
  static constexpr int BAR_BYTES = 256;
  static constexpr int PARAM_FLOATS = 3 * BN;
  // pooling: CHUNK_W accumulator columns of every tile row, as [CHUNK_W / 32][128][33] (conflict-free column reads)
  static constexpr int CHUNK_W = 64;
  static constexpr int CHUNK_FLOATS = CHUNK_W / 32 * TC_BM * 33;
  // TC_POOL: row weights [128][4] + cross-row-group staging [4][2][8][32]; TC_MAXPOOL3: staging [4][2][2][32]
  __host__ __device__ static constexpr int extra_floats(int epi) { return epi == TC_POOL ? 128 * 4 + 4 * 2 * 8 * 32 : (epi == TC_MAXPOOL3 ? 4 * 2 * 2 * 32 : 0); }
  __host__ __device__ static constexpr int consumer_floats(int epi) { return PARAM_FLOATS + (tc_pooling(epi) ? CHUNK_FLOATS + extra_floats(epi) : 0); }
  // Conv2d: the finished accumulator, one float32 row per tile row (+4 floats: 128-bit row reads without bank conflicts)
  static constexpr int ACC_LD = BN + 4;
  // box epilogues: 16 KB boxes of 128 rows x 128 bytes, float32 [BN / 32] or hi [BN / 64] then lo [BN / 64]
  static constexpr int BOX_BYTES = TC_BM * 128;
  __host__ __device__ static constexpr int stage_tile_bytes(int epi) {
    return tc_pooling(epi) ? 0 : (epi == TC_CONV2D ? TC_BM * ACC_LD * 4 : TC_BM * BN * 4);
  }
  __host__ __device__ static constexpr int total(int epi, int op_bytes = NSTAGE * STAGE_BYTES) {
    return op_bytes + stage_tile_bytes(epi) + BAR_BYTES + 2 * consumer_floats(epi) * 4 + 1024;   // + alignment slack
  }
};
static_assert(TcSmem<128>::total(TC_POOL) <= TC_SMEM_MAX && TcSmem<64>::total(TC_MAXPOOL3) <= TC_SMEM_MAX &&
              TcSmem<128>::total(TC_CONV2D) <= TC_SMEM_MAX && TcSmem<64>::total(TC_CONV2D) <= TC_SMEM_MAX &&
              TcSmem<32>::total(TC_CONV2D) <= TC_SMEM_MAX && TcSmem<128>::total(TC_BIAS_F32) <= TC_SMEM_MAX,
              "gemm_tc: shared memory");

// Per-column parameters of the element-wise epilogues (bias | bn_scale | bn_shift) of the tile at column n0, staged by the
// 128 threads of a consumer warpgroup.  With a single column tile they are the same for every tile of the warpgroup: staged
// once.
template <int BN, int EPI>
__device__ __forceinline__ void tc_stage_params(const TcArgs& a, float* params, int bar, int n0, int et) {
  named_sync(bar, 128);
  for (int i = et; i < BN; i += 128) {
    const int n = n0 + i;
    const bool ok = n < a.N;
    params[i] = (ok && a.bias) ? a.bias[n] : 0.f;
    constexpr bool has_bn = EPI != TC_BIAS_F32;
    params[BN + i] = (ok && has_bn) ? a.bn_scale[n] * (EPI == TC_CONV2D ? a.acc_scale : 1.f) : 1.f;   // (2^-k: exact)
    params[2 * BN + i] = (ok && has_bn) ? a.bn_shift[n] : 0.f;
  }
  named_sync(bar, 128);
}

// ------------------------------------------------------------------------------------ the box epilogue of one 128-row tile
// bias -> float32 rows, or bias -> LeakyReLU -> BatchNorm affine -> float32 rows / hi/lo planes, applied to the accumulator
// fragments of the 128 threads of a consumer warpgroup and written into the 128B-swizzled boxes of `tile`.
// Fragment (tc_ptx.cuh): acc[h][4 j + e] is row 64 h + 16 quad + lane / 4 + 8 (e / 2), column 8 j + 2 (lane % 4) + e % 2.
// 128B swizzle: the 16-byte chunk q of box row r sits at chunk q ^ (r % 8), and r % 8 = lane / 4 for every row of a thread.
// A warp's stores of one (h, e / 2, j) cover 8 rows x 32 bytes (float32) or 8 rows x 16 bytes per plane: no bank conflicts
// beyond the minimum wavefronts.
template <int BN, int EPI>
__device__ __forceinline__ void tc_box_epilogue(const TcArgs& a, const float* params, float (&acc)[2][BN / 2],
                                                uint32_t tile, int quad, int lane) {
  using S = TcSmem<BN>;
  const int r0 = 16 * quad + (lane >> 2), sw = lane >> 2, cq = lane & 3;
#pragma unroll
  for (int j = 0; j < BN / 8; j++) {
    const int col = 8 * j + 2 * cq;
    const float2 bias = *reinterpret_cast<const float2*>(params + col);
    float2 bsc = make_float2(1.f, 1.f), bsh = make_float2(0.f, 0.f);
    if (EPI != TC_BIAS_F32) {
      bsc = *reinterpret_cast<const float2*>(params + BN + col);
      bsh = *reinterpret_cast<const float2*>(params + 2 * BN + col);
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
#pragma unroll
      for (int e2 = 0; e2 < 2; e2++) {
        const int row = 64 * h + r0 + 8 * e2;
        float x0 = fmaf(acc[h][4 * j + 2 * e2], a.acc_scale, bias.x);
        float x1 = fmaf(acc[h][4 * j + 2 * e2 + 1], a.acc_scale, bias.y);
        if (EPI != TC_BIAS_F32) {
          x0 = fmaf(leaky(x0), bsc.x, bsh.x);
          x1 = fmaf(leaky(x1), bsc.y, bsh.y);
        }
        if (EPI == TC_LEAKY_BN_SPLIT) {
          // box j / 8 of each plane (64 columns), row bytes 16 (j % 8) + 4 cq
          uint16_t h0, l0, h1, l1;
          split_h16(x0, h0, l0);
          split_h16(x1, h1, l1);
          const int off = (j / 8) * S::BOX_BYTES + row * 128 + (((j & 7) ^ sw) << 4) + 4 * cq;
          st_shared_u32(tile + off, pack_u16x2(h0, h1));
          st_shared_u32(tile + (BN / 64) * S::BOX_BYTES + off, pack_u16x2(l0, l1));
        } else {
          // box j / 4 (32 columns), row bytes 32 (j % 4) + 8 cq
          const int q = 2 * (j & 3) + (cq >> 1);
          const int off = (j / 4) * S::BOX_BYTES + row * 128 + ((q ^ sw) << 4) + 8 * (cq & 1);
          st_shared_v2(tile + off, x0, x1);
        }
      }
    }
  }
}

// 32 consecutive accumulator columns of this thread's row
__device__ __forceinline__ void acc_ld32(const float* p, uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float4 v = reinterpret_cast<const float4*>(p)[i];
    r[4 * i] = __float_as_uint(v.x);
    r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z);
    r[4 * i + 3] = __float_as_uint(v.w);
  }
}

// ------------------------------------------------------------------------------------ the Conv2d epilogue of one 128-row tile
// Executed by the 128 threads of a consumer warpgroup; thread et = 32 quad + lane owns row et of the tile.  `mt` = index
// of the 128-row tile (rows mt * 128 ..), `acc_row` = this thread's row of the finished accumulator in shared memory.
template <int BN>
__device__ __forceinline__ void tc_conv2d_epilogue_tile(const TcArgs& a, const float* params, const float* acc_row,
                                                        long long mt, int n0, int quad, int lane) {
    const long long m = mt * TC_BM + quad * 32 + lane;
    // output position of this row
    long long mo = m;                 // output row
    bool row_ok = m < a.M;
    {
      const unsigned mu = (unsigned)m, per = (unsigned)(a.Wp * a.Hp);     // (the launcher checks M < 2^31)
      const unsigned item = mu / per, rem = mu - item * per;
      const int w = (int)(rem / (unsigned)a.Hp), h = (int)(rem - (unsigned)w * (unsigned)a.Hp);
      row_ok = row_ok && w >= 1 && w <= a.Wp - 2 && h >= 1 && h <= a.Hp - 2;     // a centre inside the un-padded map
      if (a.stride2) {
        row_ok = row_ok && (w & 1) && (h & 1);
        mo = ((long long)item * a.Wop + ((w - 1) >> 1) + 1) * a.Hop + ((h - 1) >> 1) + 1;
      }
    }
#pragma unroll 1
    for (int c = 0; c < BN; c += 32) {
      uint32_t r[32];
      acc_ld32(acc_row + c, r);
      if (n0 + c >= a.N) continue;
      float v[32];
      // BatchNorm2d(eval) affine -> (+ residual) -> ReLU
#pragma unroll
      for (int i = 0; i < 32; i++) v[i] = fmaf(__uint_as_float(r[i]), params[BN + c + i], params[2 * BN + c + i]);
      if (row_ok && a.res_hi) {
        const uint4* rh = reinterpret_cast<const uint4*>(a.res_hi + mo * a.ldc + n0 + c);
        const uint4* rl = reinterpret_cast<const uint4*>(a.res_lo + mo * a.ldc + n0 + c);
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const uint4 hq = rh[q], lq = rl[q];
          const uint32_t hw[4] = {hq.x, hq.y, hq.z, hq.w}, lw[4] = {lq.x, lq.y, lq.z, lq.w};
#pragma unroll
          for (int e = 0; e < 4; e++) {
            v[8 * q + 2 * e] += h16_to_f32((uint16_t)(hw[e] & 0xFFFFu)) + h16_to_f32((uint16_t)(lw[e] & 0xFFFFu));
            v[8 * q + 2 * e + 1] += h16_to_f32((uint16_t)(hw[e] >> 16)) + h16_to_f32((uint16_t)(lw[e] >> 16));
          }
        }
      }
      if (a.relu) {
#pragma unroll
        for (int i = 0; i < 32; i++) v[i] = fmaxf(v[i], 0.f);
      }
      if (row_ok) {
        if (a.out_f32) {
          float* po = a.out_f32 + mo * a.ldc + n0 + c;
#pragma unroll
          for (int i = 0; i < 8; i++)
            reinterpret_cast<float4*>(po)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
        }
        if (a.out_hi) {
          uint32_t hi[16], lo[16];
#pragma unroll
          for (int i = 0; i < 16; i++) {
            uint16_t h0, l0, h1, l1;
            split_h16(v[2 * i], h0, l0);
            split_h16(v[2 * i + 1], h1, l1);
            hi[i] = pack_u16x2(h0, h1);
            lo[i] = pack_u16x2(l0, l1);
          }
          uint4* ph = reinterpret_cast<uint4*>(a.out_hi + mo * a.ldc + n0 + c);
          uint4* pl = reinterpret_cast<uint4*>(a.out_lo + mo * a.ldc + n0 + c);
#pragma unroll
          for (int i = 0; i < 4; i++) {
            ph[i] = make_uint4(hi[4 * i], hi[4 * i + 1], hi[4 * i + 2], hi[4 * i + 3]);
            pl[i] = make_uint4(lo[4 * i], lo[4 * i + 1], lo[4 * i + 2], lo[4 * i + 3]);
          }
        }
      }
    }
}

// ------------------------------------------------------------------------------------ MaxPool1d(3) of 32 columns of a tile
// bias + MaxPool1d(3) over the rows of the m-tile `mt` (tile_rows / 3 windows of three rows), and the InstanceNorm partial
// sums of the pooled values, split at `brow3` between the tile's two items.  `dsm` = the tile's 32 accumulator columns
// [row][33] after the weight scale, `bias_c` = theirs, `nc` = the first one's output channel, `stg` = [rg 4][item 2][2][32].
// Executed by the 128 threads of a consumer warpgroup: thread (rg, col) = (et / 32, et % 32) pools windows rg, rg + 4, ...
// of column col; `bar` = the warpgroup's named barrier.  Ends with a barrier: dsm and stg may be rewritten.
// STG_IN_DSM: stg may overlap dsm (one more barrier: every thread is past its reads of dsm before stg is written).
template <bool STG_IN_DSM = false>
__device__ __forceinline__ void tc_maxpool3_cols(const TcArgs& a, const float* dsm, float* stg, const float* bias_c,
                                                 long long mt, int nc, int et, int bar) {
  {
    const int col = et & 31, rg = et >> 5, n = nc + col;
    const long long first = mt * (long long)a.tile_rows;                  // first un-pooled row of the tile
    const long long item0 = first / a.pool_item_rows;
    const long long nxt = (item0 + 1) * a.pool_item_rows;
    const int brow3 = nxt - first < a.tile_rows ? (int)(nxt - first) / 3 : a.tile_rows / 3;   // first window of the next item
    const long long p_first = first / 3;                                  // first pooled row of the tile
    const int f0 = (int)(p_first - item0 * (a.pool_item_rows / 3));       // its frame index inside item0
    const long long Mp = a.M / 3;
    const float bias = bias_c[col];
    // the sums are taken around the pooled value of the item's first window in the tile (`piv`)
    auto pooled = [&](int pr) {
      return fmaxf(fmaxf(dsm[(3 * pr) * 33 + col], dsm[(3 * pr + 1) * 33 + col]), dsm[(3 * pr + 2) * 33 + col]);
    };
    const float piv0 = pooled(0), piv1 = pooled(brow3 < a.tile_rows / 3 ? brow3 : 0);
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
    for (int pr = rg; pr < a.tile_rows / 3; pr += 4) {
      const float v = pooled(pr);
      const int sg = pr >= brow3 ? 1 : 0;
      const int frame = sg ? pr - brow3 : f0 + pr;
      const long long P = p_first + pr;
      if (P < Mp) {
        if (n < a.N) a.out_f32[P * a.ldc + n] = v + bias;
        if (frame < a.pool3_T) {
          const float dv = v - (sg ? piv1 : piv0);
          s1[sg] += dv;
          s2[sg] = fmaf(dv, dv, s2[sg]);
        }
      }
    }
    if (STG_IN_DSM) named_sync(bar, 128);
#pragma unroll
    for (int sg = 0; sg < 2; sg++) {
      stg[((rg * 2 + sg) * 2 + 0) * 32 + col] = s1[sg];
      stg[((rg * 2 + sg) * 2 + 1) * 32 + col] = s2[sg];
    }
    if (rg == 0 && n < a.N)
#pragma unroll
      for (int sg = 0; sg < 2; sg++) a.pool_part[(((size_t)mt * 2 + sg) * TC_POOL3_SLOTS + 2) * a.N + n] = sg ? piv1 : piv0;
  }
  named_sync(bar, 128);
  {   // 2 items x 2 sums x 32 columns = 128 values, one per thread: the four row groups in a fixed order
    const int col = et & 31, q = et >> 5, sg = q >> 1, j = q & 1, n = nc + col;
    const float tot = ((stg[((0 * 2 + sg) * 2 + j) * 32 + col] + stg[((1 * 2 + sg) * 2 + j) * 32 + col]) +
                       stg[((2 * 2 + sg) * 2 + j) * 32 + col]) + stg[((3 * 2 + sg) * 2 + j) * 32 + col];
    if (n < a.N) a.pool_part[(((size_t)mt * 2 + sg) * TC_POOL3_SLOTS + j) * a.N + n] = tot;
  }
  named_sync(bar, 128);     // stg and dsm are rewritten next
}

// ------------------------------------------------------------------------------------ the pooling epilogue of one 128-row tile
// Executed by the 128 threads of a consumer warpgroup; thread et = 32 quad + lane owns row et of the tile.  `mt` = index
// of the 128-row tile (rows mt * 128 ..), `acc` = the finished accumulator in registers, `bar` = the warpgroup's named
// barrier.
template <int BN, int EPI>
__device__ __forceinline__ void tc_pool_epilogue_tile(const TcArgs& a, float* params, float* chunk, float* pool_stage,
                                                 const float (&acc)[2][BN / 2], int bar, long long mt, int n0, int quad,
                                                 int lane, int et, bool stage_params) {
    const long long m = mt * (EPI == TC_MAXPOOL3 ? a.tile_rows : TC_BM) + quad * 32 + lane;
    // stage the per-column parameters of this tile; with a single column tile they are the same for every tile of this
    // warpgroup: staged once
    if (stage_params) {
      named_sync(bar, 128);
      for (int i = et; i < BN; i += 128) {
        const int n = n0 + i;
        const bool ok = n < a.N;
        params[i] = (ok && a.bias) ? a.bias[n] : 0.f;
        constexpr bool has_bn = EPI != TC_BIAS_F32 && EPI != TC_MAXPOOL3;
        params[BN + i] = (ok && has_bn) ? a.bn_scale[n] : 1.f;
        params[2 * BN + i] = (ok && has_bn) ? a.bn_shift[n] : 0.f;
      }
      named_sync(bar, 128);
    }
    // TC_POOL: the rows' pooling weights go to shared memory; `brow` = first row of the tile that belongs to the NEXT item
    // (a 128-row tile covers at most two items)
    int brow = TC_BM, valid0 = 0, valid1 = 0;   // TC_POOL: valid rows of the tile's two items ([0, valid0), [brow, brow + valid1))
    if (EPI == TC_POOL) {
      float4 pw = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < a.M) pw = *reinterpret_cast<const float4*>(a.pool_w + m * 4);
      reinterpret_cast<float4*>(pool_stage)[quad * 32 + lane] = pw;     // row of the tile
      const long long first = (long long)mt * TC_BM;
      const long long nxt = (first / a.pool_item_rows + 1) * a.pool_item_rows;
      brow = nxt - first < TC_BM ? (int)(nxt - first) : TC_BM;
      valid0 = min(brow, max(0, a.pool_T - (a.pool_item_rows - (int)(nxt - first))));
      valid1 = max(0, min(TC_BM - brow, a.pool_T));
      named_sync(bar, 128);
    }
    // accumulator fragment of this thread (tc_ptx.cuh): acc[h][4 j + e] is row 64 h + 16 quad + lane / 4 + 8 (e / 2),
    // column 8 j + 2 (lane % 4) + e % 2.  The tile goes through shared memory CW columns at a time (the registers of a
    // staged chunk are free for the reductions), which run 32 columns at a time.
    constexpr int CW = TcSmem<BN>::CHUNK_W;
    const int fr0 = 16 * quad + (lane >> 2), fc0 = 2 * (lane & 3);
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += CW) {
      {
        // every thread is past its reads of the previous chunk (the closing barrier of its last 32 columns)
#pragma unroll
        for (int c = c0; c < c0 + CW; c += 32) {
          float* dsm = chunk + (c - c0) / 32 * (128 * 33);   // [128][33]
#pragma unroll
          for (int jj = 0; jj < 4; jj++) {
#pragma unroll
            for (int e1 = 0; e1 < 2; e1++) {
              const int col = 8 * jj + fc0 + e1;
              float bb = 0.f, ss = 0.f, hh = 0.f;
              if (EPI == TC_POOL) bb = params[c + col], ss = params[BN + c + col], hh = params[2 * BN + c + col];
#pragma unroll
              for (int h = 0; h < 2; h++) {
#pragma unroll
                for (int e2 = 0; e2 < 2; e2++) {   // (MAXPOOL3: rows past tile_rows are not read)
                  const float y = acc[h][4 * (c / 8 + jj) + 2 * e2 + e1];
                  float* d = dsm + (64 * h + fr0 + 8 * e2) * 33 + col;
                  if (EPI == TC_POOL) {
                    // bias -> LeakyReLU -> BatchNorm affine, then the deviation from the per-channel pivot (the BatchNorm shift)
                    const float x = leaky(fmaf(y, a.acc_scale, bb));
                    *d = fmaf(x, ss, hh) - hh;
                  } else {
                    *d = y * a.acc_scale;
                  }
                }
              }
            }
          }
        }
      }
      named_sync(bar, 128);
#pragma unroll
      for (int c = c0; c < c0 + CW; c += 32) {
        if (EPI == TC_POOL) {
          // thread (row group rg, column col) sums its 32 rows of d for the K speakers -- independent accumulators, no
          // cross-lane traffic -- split at `brow` between the tile's two items.  The sums are taken around `piv`: 0, i.e. the
          // BatchNorm shift, the channel's mean under its running statistics; but where two of the item's valid rows in the
          // tile (rows past its pool_T frames hold garbage) sit far from it next to their difference, the channel's mean is
          // not near the shift, and the pivot is their average: a mean-dominated channel loses nothing to cancellation.
          // Where the running statistics do describe the channel, the shift is a better pivot than any one row: it is the
          // channel's mean, while a row can sit several weighted deviations from a speaker's mean (the fused pooling then
          // matches the two-pass stats_pool to 2e-6 instead of 2e-5 on OSP weights).  A row pair misses a mean-dominated
          // channel only if the two rows differ by 1/8 of the mean: a spike of 125 deviations at mean / std 1000.
          const float* dsm = chunk + (c - c0) / 32 * (128 * 33);
          const float4* wsm = reinterpret_cast<const float4*>(pool_stage);
          float* stg = pool_stage + 128 * 4;          // [rg 4][item 2][8][32]
          const int col = et & 31;
          auto pivot = [&](int lo, int n) {
            if (n <= 0) return 0.f;
            const float pa = dsm[lo * 33 + col], pb = dsm[(lo + n / 2) * 33 + col];
            return fabsf(pa + pb) > 16.f * fabsf(pa - pb) ? 0.5f * (pa + pb) : 0.f;
          };
          if (c != c0) named_sync(bar, 128);   // the previous 32 columns' totals are read from stg
          {
            const int rg = et >> 5, r_lo = rg * 32, r_hi = r_lo + 32;
#pragma unroll
            for (int sg = 0; sg < 2; sg++) {
              const int lo = sg == 0 ? r_lo : max(r_lo, brow), hi = sg == 0 ? min(r_hi, brow) : r_hi;
              const float piv = sg ? pivot(brow < TC_BM ? brow : 0, valid1) : pivot(0, valid0);
              float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
              if (a.pool_K <= 3) {               // the usual three local speakers: the fourth weight is not touched
#pragma unroll 8
                for (int rr = lo; rr < hi; rr++) {
                  const float dv = dsm[rr * 33 + col] - piv;
                  const float4 w4 = wsm[rr];
                  const float a0 = w4.x * dv, a1 = w4.y * dv, a2 = w4.z * dv;
                  s1[0] += a0; s1[1] += a1; s1[2] += a2;
                  s2[0] = fmaf(a0, dv, s2[0]); s2[1] = fmaf(a1, dv, s2[1]); s2[2] = fmaf(a2, dv, s2[2]);
                }
              } else {
#pragma unroll 8
                for (int rr = lo; rr < hi; rr++) {
                  const float dv = dsm[rr * 33 + col] - piv;
                  const float4 w4 = wsm[rr];
                  const float a0 = w4.x * dv, a1 = w4.y * dv, a2 = w4.z * dv, a3 = w4.w * dv;
                  s1[0] += a0; s1[1] += a1; s1[2] += a2; s1[3] += a3;
                  s2[0] = fmaf(a0, dv, s2[0]); s2[1] = fmaf(a1, dv, s2[1]); s2[2] = fmaf(a2, dv, s2[2]); s2[3] = fmaf(a3, dv, s2[3]);
                }
              }
#pragma unroll
              for (int k = 0; k < 4; k++) {
                stg[((rg * 2 + sg) * 8 + 2 * k) * 32 + col] = s1[k];
                stg[((rg * 2 + sg) * 8 + 2 * k + 1) * 32 + col] = s2[k];
              }
            }
          }
          named_sync(bar, 128);
          // 2 items x K speakers x 2 sums x 32 columns: the four row groups' totals are added in a fixed order; slot 8 of an
          // item is its pivot
          {
            const int twoK = 2 * a.pool_K, n = n0 + c + col;
            for (int q = et >> 5; q < 2 * twoK; q += 4) {
              const int sg = q >= twoK ? 1 : 0, j = q - sg * twoK;
              const float tot = ((stg[((0 * 2 + sg) * 8 + j) * 32 + col] + stg[((1 * 2 + sg) * 8 + j) * 32 + col]) +
                                 stg[((2 * 2 + sg) * 8 + j) * 32 + col]) + stg[((3 * 2 + sg) * 8 + j) * 32 + col];
              if (n < a.N && mt < a.m_tiles) a.pool_part[(((size_t)mt * 2 + sg) * TC_POOL_SLOTS + j) * a.N + n] = tot;
            }
            if (et < 64 && n < a.N && mt < a.m_tiles) {
              const int sg = et >> 5;
              a.pool_part[(((size_t)mt * 2 + sg) * TC_POOL_SLOTS + 8) * a.N + n] = sg ? pivot(brow < TC_BM ? brow : 0, valid1)
                                                                                      : pivot(0, valid0);
            }
          }
          if (c + 32 == c0 + CW) named_sync(bar, 128);     // the chunk buffer is rewritten by the next chunk
          continue;
        }
        if (EPI == TC_MAXPOOL3) {
          tc_maxpool3_cols(a, chunk + (c - c0) / 32 * (128 * 33), pool_stage, params + c, mt, n0 + c, et, bar);
          continue;
        }
      }
    }
}

// ------------------------------------------------------------------------------------ the kernel
// Named barriers besides 0: 1 + c = the 128 threads of consumer c (epilogue staging); 3 + c = consumer c may issue its
// mainloop (256 threads: consumer c waits, the other consumer arrives once its own MMAs are issued); element-wise
// epilogues: 5 + c = consumer c may write the shared staging tile (256 threads: consumer c waits, the other consumer
// arrives once the tile has been read: by its epilogue threads (Conv2d) or by TMA (box epilogues)).
// tmC0 / tmC1: output maps of the box epilogues (float32 rows; or hi and lo planes).
// HALO: Conv1d with few input channels.  The tap-box mode loads, per k-block, the 128 rows of the tile shifted by the tap's
// offset, so every activation row crosses L2 -> SM once per tap; the halo mode loads a tile's rows m0 .. m0 + 127 +
// (KW - 1) * dil once, into the slot of the consumer that runs the tile, and points the A descriptor of each k16 step at
// its tap's first row inside the slot (tc_ptx.cuh: a descriptor may start any whole number of rows into a swizzled tile).
// The k16 steps run in the tap-box mode's order (tap outer, 16 channels inner), so the results are bit-identical.
template <int BN, int EPI, bool HALO>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo,
               const __grid_constant__ CUtensorMap tmC0, const __grid_constant__ CUtensorMap tmC1, TcArgs a) {
  using S = TcSmem<BN>;
  constexpr bool POOLING = tc_pooling(EPI);
  constexpr int NSTAGE = HALO ? S::NSTAGE_HALO : S::NSTAGE;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* ring = HALO ? smem + 2 * a.halo_bytes : smem;   // the k-block ring (halo mode: W only)
  constexpr int RING_STAGE = HALO ? S::W_STAGE_BYTES : S::STAGE_BYTES;
  unsigned char* tile_s = smem + a.op_bytes;   // element-wise: the staging tile, shared by the consumers
  uint64_t* bars = reinterpret_cast<uint64_t*>(tile_s + S::stage_tile_bytes(EPI));
  uint64_t* full = bars;                      // [NSTAGE] TMA -> MMA
  uint64_t* empty = bars + NSTAGE;            // [NSTAGE] MMA -> TMA
  uint64_t* tile_full = bars + 2 * NSTAGE;    // [2] producer -> consumer c: tile_idx[c] holds its next tile
  uint64_t* tile_empty = tile_full + 2;       // [2] consumer c -> producer: tile_idx[c] has been read
  uint64_t* halo_full = tile_empty + 2;       // [2] halo mode: TMA -> consumer c, its slot holds its tile's halo
  uint64_t* halo_empty = halo_full + 2;       // [2] consumer c -> TMA: the MMAs of its tile are complete
  volatile int* tile_idx = reinterpret_cast<volatile int*>(halo_empty + 2);   // [2]
  float* cons = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(bars) + S::BAR_BYTES);

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform
  const int wg = warp >> 2;
  const int num_tiles = a.m_tiles * a.n_tiles;
  const int kblocks = HALO ? a.wblocks : a.KW * a.cin_blocks;   // ring entries per tile
  const int halo_box = a.halo_rows * 64, halo_cb = (a.cin + 31) / 32;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; s++) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 1);
    }
    for (int c = 0; c < 2; c++) {
      mbar_init(&tile_full[c], 1);
      mbar_init(&tile_empty[c], 128);
      mbar_init(&halo_full[c], 1);
      mbar_init(&halo_empty[c], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================================== tile scheduler + TMA producer
    // the halo producer's look-ahead state needs 48 registers; the consumers then get 224 (the launch holds 384 x 168:
    // 128 x 48 + 256 x 224 fit, 128 x 48 + 256 x 232 do not and setmaxnreg.inc would wait for ever)
    setmaxnreg_dec<HALO ? 48 : 40>();
    if (threadIdx.x == 0) {
      int stage = 0, phase = 0, next = 0;
      bool halo_next = false;   // halo mode: the halo of the CTA's next tile is on its way
      // i = position in this CTA's sequence of tiles, run by consumer i % 2.  The first tile is blockIdx.x, the later ones
      // come from the counter (pooling) or follow at a stride of the grid.  Two end marks follow the last tile: -1 (its
      // consumer passes the turn on), then -2.
      for (int i = 0, tile = blockIdx.x;; i++) {
        const int c = i & 1;
        mbar_wait(&tile_empty[c], ((i >> 1) & 1) ^ 1);
        if (tile >= num_tiles) {
          tile_idx[c] = -1;
          mbar_arrive(&tile_full[c]);
          mbar_wait(&tile_empty[c ^ 1], (((i + 1) >> 1) & 1) ^ 1);
          tile_idx[c ^ 1] = -2;
          mbar_arrive(&tile_full[c ^ 1]);
          break;
        }
        tile_idx[c] = tile;
        mbar_arrive(&tile_full[c]);
        const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
        const int m0 = mt * (EPI == TC_MAXPOOL3 ? a.tile_rows : TC_BM), n0 = nt * BN;
        if constexpr (HALO) {
          // halo of the tile at row r0 into consumer cc's slot
          auto load_halo = [&](int cc, int r0) {
            unsigned char* hs = smem + cc * a.halo_bytes;
            mbar_expect_tx(&halo_full[cc], 2 * halo_cb * halo_box);
            for (int cb = 0; cb < halo_cb; cb++) {
              tma_load_2d(hs + cb * halo_box, &tmA_hi, cb * TC_BK, r0, &halo_full[cc]);
              tma_load_2d(hs + (halo_cb + cb) * halo_box, &tmA_lo, cb * TC_BK, r0, &halo_full[cc]);
            }
          };
          // this tile's halo, unless it went out during the previous tile's W loads, once consumer c's previous tile has no
          // MMA left on the slot
          if (!halo_next) {
            mbar_wait(&halo_empty[c], ((i >> 1) & 1) ^ 1);
            load_halo(c, m0);
          }
          halo_next = false;
          // The next tile's halo goes out as soon as the other consumer's slot is free (its MMAs end as this tile's begin),
          // a whole mainloop before it is needed: behind this tile's W loads it would arrive late
          next = POOLING ? (int)gridDim.x + (int)atomicAdd(&a.tile_ctr[0], 1u) : tile + (int)gridDim.x;
          const int next_m0 = next / a.n_tiles * (EPI == TC_MAXPOOL3 ? a.tile_rows : TC_BM);
          const uint32_t next_par = (((i + 1) >> 1) & 1) ^ 1;
          for (int kb = 0; kb < kblocks; kb++) {
            const long long t0 = clock64();
            for (;;) {
              if (!halo_next && next < num_tiles && mbar_test_wait(&halo_empty[c ^ 1], next_par)) {
                load_halo(c ^ 1, next_m0);
                halo_next = true;
              }
              if (mbar_test_wait(&empty[stage], phase ^ 1)) break;
              if (clock64() - t0 > 4000000000LL) __trap();
            }
            unsigned char* st = ring + stage * RING_STAGE;
            mbar_expect_tx(&full[stage], S::W_STAGE_BYTES);
            tma_load_2d(st, &tmW_hi, kb * TC_BK, n0, &full[stage]);
            tma_load_2d(st + S::W_BYTES, &tmW_lo, kb * TC_BK, n0, &full[stage]);
            if (++stage == NSTAGE) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
        for (int j = 0; j < (HALO ? 0 : a.KW); j++) {
          for (int cb = 0; cb < a.cin_blocks; cb++) {
            mbar_wait(&empty[stage], phase ^ 1);
            unsigned char* st = smem + stage * S::STAGE_BYTES;
            mbar_expect_tx(&full[stage], S::STAGE_BYTES);
            const int kcol = (j * a.cin_blocks + cb) * TC_BK;
            tma_load_2d(st, &tmA_hi, cb * TC_BK, m0 + a.tap_off[j], &full[stage]);
            tma_load_2d(st + S::A_BYTES, &tmA_lo, cb * TC_BK, m0 + a.tap_off[j], &full[stage]);
            tma_load_2d(st + 2 * S::A_BYTES, &tmW_hi, kcol, n0, &full[stage]);
            tma_load_2d(st + 2 * S::A_BYTES + S::W_BYTES, &tmW_lo, kcol, n0, &full[stage]);
            if (++stage == NSTAGE) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
        if (!HALO) next = POOLING ? (int)gridDim.x + (int)atomicAdd(&a.tile_ctr[0], 1u) : tile + (int)gridDim.x;
        tile = next;
      }
      // every CTA has taken its last tile once all have counted themselves here: the last one returns the counter to 0
      // for the next launch on this stream
      if (POOLING) {
        __threadfence();
        if (atomicAdd(&a.tile_ctr[1], 1u) == gridDim.x - 1) {
          atomicExch(&a.tile_ctr[0], 0u);
          atomicExch(&a.tile_ctr[1], 0u);
        }
      }
    }
    return;
  }
  // ===================================================================== MMA + epilogue (consumers c = 0, 1)
  setmaxnreg_inc<HALO ? 224 : 232>();
  const int c = wg - 1, quad = warp & 3, et = threadIdx.x - 128 * wg;
  float* params = cons + c * S::consumer_floats(EPI);   // bias | bn_scale | bn_shift
  float* chunk = params + S::PARAM_FLOATS;
  float* pool_stage = chunk + S::CHUNK_FLOATS;          // TC_POOL / TC_MAXPOOL3 only
  const int bar = 1 + c, turn = 3 + c, turn_other = 3 + (c ^ 1), acc_free = 5 + c, acc_free_other = 5 + (c ^ 1);
  if (c == 1) {
    named_arrive(3, 256);                               // consumer 0 issues the first mainloop
    if (!POOLING) named_arrive(5, 256);                 // and writes the accumulator tile first
  }
  for (int n = 0;; n++) {
    mbar_wait(&tile_full[c], n & 1);
    const int tile = tile_idx[c];
    mbar_arrive(&tile_empty[c]);
    // box epilogues: the parameters are staged before the mainloop, while the accumulator is not live
    if (tc_box_store(EPI) && tile >= 0 && (a.n_tiles > 1 || n == 0))
      tc_stage_params<BN, EPI>(a, params, bar, (tile - tile / a.n_tiles * a.n_tiles) * BN, et);
    named_sync(turn, 256);
    if (tile < 0) {
      if (tile == -1) {
        named_arrive(turn_other, 256);
        // the last tile's consumer has handed the staging tile to this one: take that arrival
        if (!POOLING) named_sync(acc_free, 256);
      }
      break;
    }
    const int pos = (2 * n + c) * kblocks;              // ring position of the tile's first k-block
    int stage = pos % NSTAGE, phase = (pos / NSTAGE) & 1;
    // The first wgmma of a tile ignores the accumulator's contents.  Defined anyway: an undefined accumulator is carried
    // around the tile loop by ptxas, i.e. kept live through the epilogue, where it forces spills.
    float acc[2][BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[0][i] = acc[1][i] = 0.f;
    // halo mode: the next k16 step's first channel and its tap's first row (as a byte offset into a box)
    uint32_t htap = 0;
    int hch = 0;
    if constexpr (HALO) mbar_wait(&halo_full[c], n & 1);
    const uint32_t hs = smem_u32(smem + c * a.halo_bytes);
    for (int kb = 0; kb < kblocks; kb++) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(ring + stage * RING_STAGE);
      const uint32_t sw = HALO ? sa : sa + 2 * S::A_BYTES;
      const uint64_t w_hi = wg_desc_sw64(sw), w_lo = wg_desc_sw64(sw + S::W_BYTES);
      constexpr uint64_t HALF = (uint64_t)((64 * TC_BK * 2) >> 4);   // rows 64..127 of the A tile (64-byte rows)
      wg_fence_acc(acc[0]);
      wg_fence_acc(acc[1]);
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < TC_BK / 16; ks++) {
        const uint64_t adv = (uint64_t)((ks * 32) >> 4);   // +32 bytes per 16-element k-step
        uint64_t a_hi, a_lo;
        if constexpr (HALO) {
          // k16 step 2 kb + ks = (tap, channels hch .. hch + 15), no branch: a wgmma on a divergent path makes ptxas
          // serialise them all.  With an odd number of steps per tap set (SincNet's 5 x 80 channels) the last k-block's
          // second step reads the next tap's first 16 channels against the W columns past K, which TMA fills with zeros
          const uint32_t aa = hs + (uint32_t)(hch >> 5) * halo_box + (uint32_t)(hch & 31) * 2 + htap;
          a_hi = wg_desc_sw64(aa);
          a_lo = wg_desc_sw64(aa + halo_cb * halo_box);
          hch += 16;
          const bool next_tap = hch == a.cin;   // a.dil rows further down
          hch = next_tap ? 0 : hch;
          htap += next_tap ? a.dil * 64 : 0;
        } else {
          a_hi = wg_desc_sw64(sa) + adv;
          a_lo = wg_desc_sw64(sa + S::A_BYTES) + adv;
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
          wgmma_ss<BN>(acc[h], a_lo + h * HALF, w_hi + adv, (kb | ks) != 0);
          wgmma_ss<BN>(acc[h], a_hi + h * HALF, w_lo + adv, 1);
          wgmma_ss<BN>(acc[h], a_hi + h * HALF, w_hi + adv, 1);
        }
      }
      wg_commit();
      wg_wait<1>();
      wg_fence_acc(acc[0]);
      wg_fence_acc(acc[1]);
      // the previous k-block's slot is released once its MMAs are complete (kept as `stage - 1`, not in a register of
      // its own: the consumer's registers are at the 168 of the launch while the accumulator is live)
      if (kb > 0 && et == 0) mbar_arrive(&empty[stage == 0 ? NSTAGE - 1 : stage - 1]);
      if (++stage == NSTAGE) {
        stage = 0;
        phase ^= 1;
      }
    }
    named_arrive(turn_other, 256);       // the other consumer's MMAs queue behind these while they drain
    wg_wait<0>();
    wg_fence_acc(acc[0]);
    wg_fence_acc(acc[1]);
    if (et == 0) mbar_arrive(&empty[stage == 0 ? NSTAGE - 1 : stage - 1]);
    if (HALO && et == 0) mbar_arrive(&halo_empty[c]);
    const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
    const bool stage_params = a.n_tiles > 1 || n == 0;
    if constexpr (POOLING) {
      tc_pool_epilogue_tile<BN, EPI>(a, params, chunk, pool_stage, acc, bar, mt, nt * BN, quad, lane, et, stage_params);
    } else if constexpr (EPI == TC_CONV2D) {
      // accumulator -> the shared tile, once the other consumer's epilogue has read it; fragment (tc_ptx.cuh): acc[h][4 j + e]
      // is row 64 h + 16 quad + lane / 4 + 8 (e / 2), column 8 j + 2 (lane % 4) + e % 2
      float* acc_s = reinterpret_cast<float*>(tile_s);   // [128][ACC_LD]
      named_sync(acc_free, 256);
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r0 = 64 * h + 16 * quad + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
          const int col = 8 * j + 2 * (lane & 3);
          *reinterpret_cast<float2*>(acc_s + r0 * S::ACC_LD + col) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
          *reinterpret_cast<float2*>(acc_s + (r0 + 8) * S::ACC_LD + col) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
        }
      }
      named_sync(bar, 128);
      if (stage_params) tc_stage_params<BN, EPI>(a, params, bar, nt * BN, et);
      tc_conv2d_epilogue_tile<BN>(a, params, acc_s + et * S::ACC_LD, mt, nt * BN, quad, lane);
      named_arrive(acc_free_other, 256);
    } else {
      named_sync(acc_free, 256);          // the other consumer's boxes have been read by TMA
      tc_box_epilogue<BN, EPI>(a, params, acc, smem_u32(tile_s), quad, lane);
      fence_proxy_async_smem();
      named_sync(bar, 128);
      if (et == 0) {
        const int m0 = mt * TC_BM, n0 = nt * BN;
        if (EPI == TC_LEAKY_BN_SPLIT) {
#pragma unroll
          for (int b = 0; b < BN / 64; b++) {
            if (n0 + 64 * b >= a.N) break;
            tma_store_2d(&tmC0, tile_s + b * S::BOX_BYTES, n0 + 64 * b, m0);
            tma_store_2d(&tmC1, tile_s + (BN / 64 + b) * S::BOX_BYTES, n0 + 64 * b, m0);
          }
        } else {
#pragma unroll
          for (int b = 0; b < BN / 32; b++) {
            if (n0 + 32 * b >= a.N) break;
            tma_store_2d(&tmC0, tile_s + b * S::BOX_BYTES, n0 + 32 * b, m0);
          }
        }
        bulk_commit();
        bulk_wait_read_all();
      }
      __syncwarp();
      named_arrive(acc_free_other, 256);
    }
  }
  // the global writes of this consumer's last boxes complete before the CTA exits
  if (tc_box_store(EPI) && et == 0) bulk_wait_all();
}

// ------------------------------------------------------------------------------------ the weight-stationary MaxPool3 kernel
// TC_MAXPOOL3 for Conv1d over few channels (SincNet's conv1 and conv2) with the operands swapped: D^T = W . X^T.  The A
// operand is W, its 64 (padded) output channels one m64; the B operand is the tile's halo, N = TCW_N time rows, so one MMA
// covers a tile of up to 112 rows (tile_rows = 111 for SincNet) instead of 128 for 111.  W, hi and lo, goes to shared
// memory once per CTA and stays there for every tile: nothing streams through a ring, and the producer only loads halos.
// The halo slots are the same 64B-swizzled [hi | lo][ceil(cin / 32)] boxes as in gemm_tc_kernel<.., true>, and the B
// descriptor of each k16 step starts its tap's offset rows into the slot (dg_selftest_wgmma_b_row_shift).
// Per output element the products and their order are those of gemm_tc_kernel: k16 steps tap outer, 16 channels inner,
// lo.hi, hi.lo, hi.hi per step; a K of an odd number of k16 steps runs no zero step at the end, which adds nothing.
// The accumulator fragment (tc_ptx.cuh) is transposed: acc[4 j + e] is output channel 16 quad + lane / 4 + 8 (e / 2), tile
// row 8 j + 2 (lane % 4) + e % 2.  The epilogue stages it 32 channels at a time as [row][33] and pools it with the tap-box
// kernel's code, so the pooled rows and the InstanceNorm partials are bit-identical.  Each consumer has its own staging
// chunk, so the two epilogues may run at once (the epilogue of a tile takes longer than its MMAs); to fit one per consumer
// next to 104 KB of W (conv1) and two halo slots, the cross-row-group sums are staged in the chunk itself once it has been
// read, and the bias is staged once for both.
constexpr int TCW_N = 112;
struct TcWsSmem {
  static constexpr int W_BOX = 64 * TC_BK * 2;                          // 64 channels x 32 k of one plane: 4 KB
  static constexpr int BAR_BYTES = 128;
  static constexpr int CHUNK_FLOATS = TCW_N * 33;                      // [112][33]; then the [4][2][2][32] sums
  static constexpr int STAGE_FLOATS = 64 + 2 * CHUNK_FLOATS;            // bias | consumer 0's chunk | consumer 1's chunk
  __host__ static int halo_rows(int KW, int dil) { return (TCW_N + (KW - 1) * dil + 7) / 8 * 8; }
  __host__ static int w_plane_bytes(int K) { return (K + TC_BK - 1) / TC_BK * W_BOX; }
  // [W hi][W lo][halo slot 0][halo slot 1][barriers][epilogue staging]
  __host__ static int op_bytes(int cin, int KW, int dil) {
    return 2 * w_plane_bytes(KW * cin) + 2 * TcSmem<64>::halo_bytes(cin, halo_rows(KW, dil));
  }
  __host__ static int total(int op) { return op + BAR_BYTES + STAGE_FLOATS * 4 + 1024; }   // + alignment slack
};

__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_ws_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                  const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo, TcArgs a) {
  using S = TcWsSmem;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int w_plane = a.wblocks * S::W_BOX;
  unsigned char* halo = smem + 2 * w_plane;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + a.op_bytes);
  uint64_t* w_full = bars;                    // [1] TMA -> consumers: W is resident
  uint64_t* tile_full = bars + 1;             // [2] producer -> consumer c: tile_idx[c] holds its next tile
  uint64_t* tile_empty = bars + 3;            // [2] consumer c -> producer: tile_idx[c] has been read
  uint64_t* halo_full = bars + 5;             // [2] TMA -> consumer c: its slot holds its tile's halo
  uint64_t* halo_empty = bars + 7;            // [2] consumer c -> producer: the MMAs of its tile are complete
  volatile int* tile_idx = reinterpret_cast<volatile int*>(bars + 9);   // [2]
  float* bias_s = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(bars) + S::BAR_BYTES);

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform
  const int wg = warp >> 2;
  const int num_tiles = a.m_tiles;
  const int halo_box = a.halo_rows * 64, halo_cb = (a.cin + 31) / 32;

  if (threadIdx.x == 0) {
    mbar_init(w_full, 1);
    for (int c = 0; c < 2; c++) {
      mbar_init(&tile_full[c], 1);
      mbar_init(&tile_empty[c], 128);
      mbar_init(&halo_full[c], 1);
      mbar_init(&halo_empty[c], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < 64) bias_s[threadIdx.x] = (int)threadIdx.x < a.N && a.bias ? a.bias[threadIdx.x] : 0.f;
  __syncthreads();

  if (wg == 0) {
    // ===================================================================== tile scheduler + TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(w_full, 2 * w_plane);
      for (int b = 0; b < a.wblocks; b++) {   // W columns past K are zero-filled by TMA
        tma_load_2d(smem + b * S::W_BOX, &tmW_hi, b * TC_BK, 0, w_full);
        tma_load_2d(smem + w_plane + b * S::W_BOX, &tmW_lo, b * TC_BK, 0, w_full);
      }
      // i = position in this CTA's sequence of tiles, run by consumer i % 2: the first is blockIdx.x, the later ones come
      // from the counter.  A tile's halo goes out as soon as its consumer's previous tile has no MMA left on the slot, i.e.
      // while that tile's epilogue runs.  Two end marks follow the last tile: -1 (its consumer passes the turn on), then -2.
      for (int i = 0, tile = blockIdx.x;; i++) {
        const int c = i & 1;
        if (tile < num_tiles) {
          mbar_wait(&halo_empty[c], ((i >> 1) & 1) ^ 1);
          unsigned char* hs = halo + c * a.halo_bytes;
          const int r0 = tile * a.tile_rows;
          mbar_expect_tx(&halo_full[c], 2 * halo_cb * halo_box);
          for (int cb = 0; cb < halo_cb; cb++) {
            tma_load_2d(hs + cb * halo_box, &tmA_hi, cb * TC_BK, r0, &halo_full[c]);
            tma_load_2d(hs + (halo_cb + cb) * halo_box, &tmA_lo, cb * TC_BK, r0, &halo_full[c]);
          }
        }
        mbar_wait(&tile_empty[c], ((i >> 1) & 1) ^ 1);
        if (tile >= num_tiles) {
          tile_idx[c] = -1;
          mbar_arrive(&tile_full[c]);
          mbar_wait(&tile_empty[c ^ 1], (((i + 1) >> 1) & 1) ^ 1);
          tile_idx[c ^ 1] = -2;
          mbar_arrive(&tile_full[c ^ 1]);
          break;
        }
        tile_idx[c] = tile;
        mbar_arrive(&tile_full[c]);
        tile = (int)gridDim.x + (int)atomicAdd(&a.tile_ctr[0], 1u);
      }
      // every CTA has taken its last tile once all have counted themselves here: the last one returns the counter to 0
      // for the next launch on this stream
      __threadfence();
      if (atomicAdd(&a.tile_ctr[1], 1u) == gridDim.x - 1) {
        atomicExch(&a.tile_ctr[0], 0u);
        atomicExch(&a.tile_ctr[1], 0u);
      }
    }
    return;
  }
  // ===================================================================== MMA + epilogue (consumers c = 0, 1)
  setmaxnreg_inc<232>();
  const int c = wg - 1, quad = warp & 3, et = threadIdx.x - 128 * wg;
  // named barriers besides 0: 1 + c = the 128 threads of consumer c; 3 + c = consumer c may issue its mainloop
  const int bar = 1 + c, turn = 3 + c, turn_other = 3 + (c ^ 1);
  float* chunk = bias_s + 64 + c * S::CHUNK_FLOATS;   // [TCW_N][33]: 32 accumulator channels of every tile row
  if (c == 1) named_arrive(3, 256);           // consumer 0 issues the first mainloop
  const int ksteps = a.KW * a.cin / 16;
  const uint32_t w_s = smem_u32(smem), hs = smem_u32(halo + c * a.halo_bytes);
  mbar_wait(w_full, 0);
  for (int n = 0;; n++) {
    mbar_wait(&tile_full[c], n & 1);
    const int tile = tile_idx[c];
    mbar_arrive(&tile_empty[c]);
    named_sync(turn, 256);
    if (tile < 0) {
      if (tile == -1) named_arrive(turn_other, 256);
      break;
    }
    // defined before the first wgmma, which ignores it: an undefined accumulator is kept live through the epilogue
    float acc[TCW_N / 2];
#pragma unroll
    for (int i = 0; i < TCW_N / 2; i++) acc[i] = 0.f;
    mbar_wait(&halo_full[c], n & 1);
    // the next k16 step's first channel and its tap's first row (as a byte offset into a box)
    uint32_t htap = 0;
    int hch = 0;
    wg_fence_acc(acc);
    wg_fence();
    for (int s = 0; s < ksteps; s++) {
      const uint32_t wa = w_s + (uint32_t)(s >> 1) * S::W_BOX + (uint32_t)(s & 1) * 32;
      const uint64_t w_hi = wg_desc_sw64(wa), w_lo = wg_desc_sw64(wa + w_plane);
      const uint32_t xa = hs + (uint32_t)(hch >> 5) * halo_box + (uint32_t)(hch & 31) * 2 + htap;
      const uint64_t x_hi = wg_desc_sw64(xa), x_lo = wg_desc_sw64(xa + halo_cb * halo_box);
      hch += 16;
      const bool next_tap = hch == a.cin;   // a.dil rows further down
      hch = next_tap ? 0 : hch;
      htap += next_tap ? a.dil * 64 : 0;
      wgmma_ss<TCW_N>(acc, w_hi, x_lo, s != 0);
      wgmma_ss<TCW_N>(acc, w_lo, x_hi, 1);
      wgmma_ss<TCW_N>(acc, w_hi, x_hi, 1);
    }
    wg_commit();
    named_arrive(turn_other, 256);            // the other consumer's MMAs queue behind these while they drain
    wg_wait<0>();
    wg_fence_acc(acc);
    if (et == 0) mbar_arrive(&halo_empty[c]);
    // channels c0 .. c0 + 31 are held by warps c0 / 16 and c0 / 16 + 1 of the warpgroup; `frag` = this thread's first
    // element (row 2 (lane % 4), channel 16 (quad % 2) + lane / 4) in the chunk
    const uint32_t frag = smem_u32(chunk) + 4 * (2 * (lane & 3) * 33 + 16 * (quad & 1) + (lane >> 2));
#pragma unroll
    for (int c0 = 0; c0 < 64; c0 += 32) {
      if ((quad >> 1) == (c0 >> 5)) {
#pragma unroll
        for (int j = 0; j < TCW_N / 8; j++)
#pragma unroll
          for (int e = 0; e < 4; e++)
            st_shared_u32(frag + 4 * ((8 * j + (e & 1)) * 33 + 8 * (e >> 1)), __float_as_uint(acc[4 * j + e] * a.acc_scale));
      }
      named_sync(bar, 128);
      tc_maxpool3_cols<true>(a, chunk, chunk, bias_s + c0, tile, c0, et, bar);
    }
  }
}

// ------------------------------------------------------------------------------------ host side
// 16-bit (or, `f32`, float32) matrix [rows, cols] row-major (cols contiguous, row pitch `ld` elements); box = box_cols x
// box_rows, swizzled by the box row's width (64 or 128 bytes)
static int make_map(CUtensorMap* m, const void* base, long long rows, int cols, int ld, int box_cols, int box_rows,
                    bool f32 = false) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return -2;
  }
  const int esize = f32 ? 4 : 2;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims,
                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  box_cols * esize == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
    return -2;
  }
  return 0;
}

// Tile counters of the dynamic schedule, one pair per (device, stream): launches on one stream run one after another and
// each leaves its counter at 0, launches on different streams may overlap and never share one.
constexpr int TC_CTR_SLOTS = 1024;
__device__ unsigned g_tc_tile_ctr[TC_CTR_SLOTS][2];

static unsigned* tile_counter(cudaStream_t st) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, int> slot_of;
  static int used[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    set_error("gemm_tc: no current CUDA device");
    return nullptr;
  }
  int slot;
  {
    std::lock_guard<std::mutex> lock(mu);
    auto it = slot_of.find({dev, st});
    if (it != slot_of.end()) {
      slot = it->second;
    } else {
      if (used[dev] == TC_CTR_SLOTS) {
        set_error("gemm_tc: more than " + std::to_string(TC_CTR_SLOTS) + " streams have launched GEMMs on one device");
        return nullptr;
      }
      slot = slot_of[{dev, st}] = used[dev]++;
    }
  }
  void* base = nullptr;
  if (cudaGetSymbolAddress(&base, g_tc_tile_ctr) != cudaSuccess) {
    set_error("gemm_tc: cannot address the tile counters");
    return nullptr;
  }
  return static_cast<unsigned*>(base) + 2 * slot;
}

// operand maps, output maps (box epilogues: float32 rows, or hi and lo planes, as [M, N] of pitch ldc) and kernel arguments
// of one launch; tiles of `bn` columns
// column tile width of a launch (element-wise and pooling epilogues; Conv2d picks it from Npad in launch_gemm_tc)
static int tc_bn(const TcGemm& g) { return g.epi == TC_MAXPOOL3 || (g.Npad == 64 && g.epi == TC_BIAS_F32) ? 64 : 128; }
// rows of a tile's halo: the 128 rows of the MMA and (KW - 1) * dil below them (KW * dil when K is an odd number of k16
// steps: the last one reads the first rows of a tap past the last), rounded up to whole 8-row swizzle groups
static int tc_halo_rows(const TcGemm& g) {
  return (TC_BM + (g.KW - ((g.KW * g.Cin) % 32 ? 0 : 1)) * g.dil + 7) / 8 * 8;
}
template <int BN>
static int tc_halo_smem(const TcGemm& g) { return TcSmem<BN>::total(g.epi, TcSmem<BN>::halo_op_bytes(g.Cin, tc_halo_rows(g))); }

// TC_MAXPOOL3 takes the weight-stationary kernel where its tiles fit the MMA's 112 rows and W, both halo slots and the
// epilogue's buffers fit in shared memory (SincNet's conv1: 104 KB of W, 2 x 45 KB of halo)
bool gemm_tc_ws(const TcGemm& g) {
  if (g.epi != TC_MAXPOOL3 || g.tap_boxes || g.tap_off || g.KW < 2 || g.dil < 1 || g.Cin % 16 || g.Cin > 128 ||
      g.pool3_tile_rows > TCW_N || TcWsSmem::halo_rows(g.KW, g.dil) > 256)
    return false;
  return TcWsSmem::total(TcWsSmem::op_bytes(g.Cin, g.KW, g.dil)) <= TC_SMEM_MAX;
}

// The halo mode is taken by every Conv1d with several taps over at most 128 channels (a multiple of 16) whose halo is one
// TMA box (at most 256 rows) and fits, with the W ring and the epilogue's buffers, in shared memory
bool gemm_tc_halo(const TcGemm& g) {
  if (g.tap_boxes || g.epi == TC_CONV2D || g.tap_off || g.KW < 2 || g.dil < 1 || g.Cin % 16 || g.Cin > 128 ||
      tc_halo_rows(g) > 256)
    return false;
  return gemm_tc_ws(g) || (tc_bn(g) == 64 ? tc_halo_smem<64>(g) : tc_halo_smem<128>(g)) <= TC_SMEM_MAX;
}

static int tc_setup(const TcGemm& g, int bn, int epi, bool halo, CUtensorMap* maps, TcArgs& a, bool ws = false) {
  const int Ktot = g.KW * g.Cin, bk = TC_BK, a_rows = ws ? TcWsSmem::halo_rows(g.KW, g.dil) : (halo ? tc_halo_rows(g) : TC_BM);
  if (make_map(&maps[0], g.A_hi, g.Mtot, g.Cin, g.lda, bk, a_rows) || make_map(&maps[1], g.A_lo, g.Mtot, g.Cin, g.lda, bk, a_rows) ||
      make_map(&maps[2], g.W_hi, g.Npad, Ktot, Ktot, bk, bn) || make_map(&maps[3], g.W_lo, g.Npad, Ktot, Ktot, bk, bn))
    return -2;
  memset(&maps[4], 0, 2 * sizeof(CUtensorMap));
  if (epi == TC_LEAKY_BN_SPLIT) {
    if (make_map(&maps[4], g.out_hi, g.M, g.N, g.ldc, 64, TC_BM) || make_map(&maps[5], g.out_lo, g.M, g.N, g.ldc, 64, TC_BM))
      return -2;
  } else if (tc_box_store(epi)) {
    if (make_map(&maps[4], g.out_f32, g.M, g.N, g.ldc, 32, TC_BM, true)) return -2;
  }
  a = TcArgs{};
  a.M = g.M; a.N = g.N; a.n_tiles = (g.N + bn - 1) / bn;
  a.tile_rows = epi == TC_MAXPOOL3 ? g.pool3_tile_rows : TC_BM;
  a.pool3_T = g.pool3_T;
  a.m_tiles = (int)((g.M + a.tile_rows - 1) / a.tile_rows);
  a.KW = g.KW; a.dil = g.dil; a.cin_blocks = g.Cin / bk;
  a.bias = g.bias; a.bn_scale = g.bn_scale; a.bn_shift = g.bn_shift;
  a.out_f32 = g.out_f32; a.out_hi = reinterpret_cast<__nv_bfloat16*>(g.out_hi);
  a.out_lo = reinterpret_cast<__nv_bfloat16*>(g.out_lo); a.ldc = g.ldc;
  a.acc_scale = g.w_scale > 0.f ? 1.f / g.w_scale : 1.f;
  for (int j = 0; j < 9; j++) a.tap_off[j] = j < g.KW ? (g.tap_off ? g.tap_off[j] : j * g.dil) : 0;
  a.Wp = g.Wp; a.Hp = g.Hp; a.Wop = g.Wop; a.Hop = g.Hop; a.stride2 = g.stride2; a.relu = g.relu;
  a.res_hi = reinterpret_cast<const __nv_bfloat16*>(g.res_hi);
  a.res_lo = reinterpret_cast<const __nv_bfloat16*>(g.res_lo);
  a.pool_w = g.pool_w; a.pool_part = g.pool_part; a.pool_item_rows = g.pool_item_rows; a.pool_K = g.pool_K; a.pool_T = g.pool_T;
  a.cin = g.Cin;
  if (ws) {
    a.halo_rows = a_rows;
    a.wblocks = (Ktot + bk - 1) / bk;
    a.halo_bytes = TcSmem<64>::halo_bytes(g.Cin, a_rows);
    a.op_bytes = TcWsSmem::op_bytes(g.Cin, g.KW, g.dil);
  } else if (halo) {
    a.halo_rows = a_rows;
    a.wblocks = (Ktot + bk - 1) / bk;     // W columns past Ktot of the last k-block are zero-filled by TMA
    a.halo_bytes = bn == 64 ? TcSmem<64>::halo_bytes(g.Cin, a_rows) : TcSmem<128>::halo_bytes(g.Cin, a_rows);
    a.op_bytes = bn == 64 ? TcSmem<64>::halo_op_bytes(g.Cin, a_rows) : TcSmem<128>::halo_op_bytes(g.Cin, a_rows);
  } else {
    a.op_bytes = bn == 128 ? TcSmem<128>::NSTAGE * TcSmem<128>::STAGE_BYTES
                           : (bn == 64 ? TcSmem<64>::NSTAGE * TcSmem<64>::STAGE_BYTES : TcSmem<32>::NSTAGE * TcSmem<32>::STAGE_BYTES);
  }
  return 0;
}

static int tc_grid(const TcArgs& a) {
  const int sms = usable_sms();
  const int tiles = a.m_tiles * a.n_tiles;
  return tiles < sms ? tiles : sms;
}

template <int BN, int EPI, bool HALO>
static int launch_tc(const TcGemm& g, cudaStream_t st) {
  using S = TcSmem<BN>;
  CUtensorMap m[6];
  TcArgs a;
  if (tc_setup(g, BN, EPI, HALO, m, a)) return -2;
  if (tc_pooling(EPI) && !(a.tile_ctr = tile_counter(st))) return -2;
  auto kern = gemm_tc_kernel<BN, EPI, HALO>;
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done))   // halo mode: the size depends on the shape
    DG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, HALO ? TC_SMEM_MAX : S::total(EPI)));
  kern<<<tc_grid(a), TC_THREADS, S::total(EPI, a.op_bytes), st>>>(m[0], m[1], m[2], m[3], m[4], m[5], a);
  DG_LAUNCHED();
  return 0;
}

static int launch_tc_ws(const TcGemm& g, cudaStream_t st) {
  CUtensorMap m[6];
  TcArgs a;
  if (tc_setup(g, 64, TC_MAXPOOL3, true, m, a, true) || !(a.tile_ctr = tile_counter(st))) return -2;
  static bool attr_done[64] = {};
  if (first_use_on_device(attr_done))   // the size depends on the shape
    DG_CUDA(cudaFuncSetAttribute(gemm_tc_ws_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX));
  gemm_tc_ws_kernel<<<tc_grid(a), TC_THREADS, TcWsSmem::total(a.op_bytes), st>>>(m[0], m[1], m[2], m[3], a);
  DG_LAUNCHED();
  return 0;
}

template <int BN, int EPI>
static int launch_tc(const TcGemm& g, cudaStream_t st) {
  return gemm_tc_halo(g) ? launch_tc<BN, EPI, true>(g, st) : launch_tc<BN, EPI, false>(g, st);
}

int launch_gemm_tc(const TcGemm& g, cudaStream_t st) {
  ProfScope _ps(g.tag ? g.tag : "gemm_tc", st);
  if (g.Cin % (gemm_tc_halo(g) ? 16 : 64) || g.lda % 8 || g.ldc % (g.epi == TC_LEAKY_BN_SPLIT ? 8 : 4) ||
      (g.Npad % 128 && g.Npad != 64 && g.Npad != 32) || g.KW < 1 || g.KW > 9) {
    set_error("gemm_tc: Cin must be a multiple of 64 (a Conv1d of 2..9 taps over at most 128 channels whose tile halo fits "
              "in shared memory, e.g. Cin 80: a multiple of 16), A pitch a multiple of 8, output pitch a multiple of 4 "
              "(8 for 16-bit planes), padded N 32, 64 or a multiple of 128, at most 9 taps");
    return -1;
  }
  if (g.epi == TC_LEAKY_BN_SPLIT && g.N % 32) {
    set_error("gemm_tc (planes): N must be a multiple of 32");
    return -1;
  }
  if (tc_box_store(g.epi)) {
    // TMA stores: 16-byte aligned base and pitch, row coordinates below 2^31
    const bool planes = g.epi == TC_LEAKY_BN_SPLIT;
    const uintptr_t base = planes ? ((uintptr_t)g.out_hi | (uintptr_t)g.out_lo) : (uintptr_t)g.out_f32;
    if (!base || (planes && (!g.out_hi || !g.out_lo)) || base % 16 || g.ldc < g.N || g.M >= (1LL << 31)) {
      set_error("gemm_tc: the output needs a 16-byte aligned base, a pitch of at least N and fewer than 2^31 rows");
      return -1;
    }
  }
  if (g.epi == TC_CONV2D) {
    if (g.ldc % 32 || g.N % 32 || g.Wp < 3 || g.Hp < 3 || (!g.out_hi && !g.out_f32) || g.M >= (1LL << 31)) {
      set_error("gemm_tc (conv2d): channel counts must be multiples of 32");
      return -1;
    }
    if (g.Npad == 32) return launch_tc<32, TC_CONV2D, false>(g, st);
    if (g.Npad == 64) return launch_tc<64, TC_CONV2D, false>(g, st);
    return launch_tc<128, TC_CONV2D, false>(g, st);
  }
  if (g.epi == TC_POOL) {
    if (g.Npad % 128 || !g.pool_w || !g.pool_part || g.pool_K < 1 || g.pool_K > 4 || g.pool_item_rows < TC_BM || g.pool_T < 1 ||
        g.pool_T > g.pool_item_rows) {
      set_error("gemm_tc (pool): needs 128-wide tiles, 1..4 speakers, items of at least 128 rows and 1..item rows valid frames");
      return -1;
    }
    return launch_tc<128, TC_POOL>(g, st);
  }
  if (g.epi == TC_MAXPOOL3) {
    if (g.Npad != 64 || !g.out_f32 || !g.pool_part || g.pool3_T < 1 || g.pool3_tile_rows < 3 || g.pool3_tile_rows > 126 ||
        g.pool3_tile_rows % 3 || g.pool_item_rows % g.pool3_tile_rows || g.M % g.pool_item_rows) {
      set_error("gemm_tc (maxpool3): needs 64 output channels and tiles of 3..126 rows (a multiple of 3) that divide the item");
      return -1;
    }
    if (gemm_tc_ws(g)) return launch_tc_ws(g, st);
    return launch_tc<64, TC_MAXPOOL3>(g, st);
  }
  if (g.Npad == 64 && g.epi == TC_BIAS_F32) return launch_tc<64, TC_BIAS_F32>(g, st);
  switch (g.epi) {
    case TC_BIAS_F32:
      return launch_tc<128, TC_BIAS_F32>(g, st);
    case TC_LEAKY_BN_SPLIT:
      return launch_tc<128, TC_LEAKY_BN_SPLIT>(g, st);
    default:
      return launch_tc<128, TC_LEAKY_BN_F32>(g, st);
  }
}

// ------------------------------------------------------------------------------------ descriptor row-shift probe
// One warpgroup TMA-loads A and B (32 fp16 channels per row) with the 64B swizzle of the GEMM's operand boxes and, for every
// shift r = 0..8 and k16 step ks, runs one m64nBNk16 product whose SHIFT_B operand descriptor starts r rows into its tile:
// A rows r..r+63 with B's 8 rows (m64n8), or A's 64 rows with B rows r..r+63 (m64n64); out[r][ks][64][BN].
// base_offset_mode 1 also sets the shifted descriptor's matrix base offset field (bits 49-51) to (start address >> 7) & 7.
template <bool SHIFT_B>
struct RowShiftProbe {
  static constexpr int BN = SHIFT_B ? 64 : 8, A_ROWS = SHIFT_B ? 64 : 72, B_ROWS = SHIFT_B ? 72 : 8;
};

template <bool SHIFT_B>
__global__ void __launch_bounds__(128) wgmma_row_shift_kernel(const __grid_constant__ CUtensorMap tmA,
                                                              const __grid_constant__ CUtensorMap tmB, int base_offset_mode,
                                                              float* out) {
  using P = RowShiftProbe<SHIFT_B>;
  __shared__ __align__(1024) unsigned char sm[(P::A_ROWS + P::B_ROWS) * 64];
  __shared__ uint64_t bar;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, sizeof(sm));
    tma_load_2d(sm, &tmA, 0, 0, &bar);
    tma_load_2d(sm + P::A_ROWS * 64, &tmB, 0, 0, &bar);
  }
  mbar_wait(&bar, 0);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  for (int r = 0; r <= 8; r++) {
    for (int ks = 0; ks < 2; ks++) {
      const uint32_t sa = smem_u32(sm) + (SHIFT_B ? 0 : r * 64) + ks * 32;
      const uint32_t sb = smem_u32(sm + P::A_ROWS * 64) + (SHIFT_B ? r * 64 : 0) + ks * 32;
      const uint64_t base = base_offset_mode ? (uint64_t)(((SHIFT_B ? sb : sa) >> 7) & 7) << 49 : 0;
      const uint64_t da = wg_desc_sw64(sa) | (SHIFT_B ? 0 : base), db = wg_desc_sw64(sb) | (SHIFT_B ? base : 0);
      float d[P::BN / 2];
      for (int i = 0; i < P::BN / 2; i++) d[i] = 0.f;
      wg_fence_acc(d);
      wg_fence();
      wgmma_ss<P::BN>(d, da, db, 0);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(d);
      for (int i = 0; i < P::BN / 2; i++)
        out[((r * 2 + ks) * 64 + 16 * w + l / 4 + 8 * ((i / 2) % 2)) * P::BN + 8 * (i / 4) + 2 * (l % 4) + i % 2] = d[i];
    }
  }
}

template <bool SHIFT_B>
static int selftest_row_shift(int base_offset_mode, unsigned* ok_shifts) {
  using P = RowShiftProbe<SHIFT_B>;
  // small integers: every product and sum is exact in fp16 inputs and the float32 accumulator
  std::vector<float> Af(P::A_ROWS * 32), Bf(P::B_ROWS * 32);
  std::vector<float>& shifted = SHIFT_B ? Bf : Af;
  std::vector<float>& fixed = SHIFT_B ? Af : Bf;
  for (size_t i = 0; i < shifted.size(); i++) shifted[i] = (float)((int)((i * 7 + i / 32 * 3) % 9) - 4);
  for (size_t i = 0; i < fixed.size(); i++) fixed[i] = (float)((int)((i * 5 + i / 32) % 7) - 3);
  std::vector<uint16_t> A(Af.size()), B(Bf.size());
  for (size_t i = 0; i < A.size(); i++) A[i] = host_f32_to_h16(Af[i]);
  for (size_t i = 0; i < B.size(); i++) B[i] = host_f32_to_h16(Bf[i]);
  std::vector<float> out(9 * 2 * 64 * P::BN);
  DevBuf dA, dB, dO;
  CUtensorMap mA, mB;
  if (upload_u16(dA, A) || upload_u16(dB, B) || dO.ensure(out.size() * 4) ||
      make_map(&mA, dA.p, P::A_ROWS, 32, 32, 32, P::A_ROWS) || make_map(&mB, dB.p, P::B_ROWS, 32, 32, 32, P::B_ROWS))
    return -2;
  wgmma_row_shift_kernel<SHIFT_B><<<1, 128>>>(mA, mB, base_offset_mode, dO.as<float>());
  DG_CUDA(cudaGetLastError());
  DG_CUDA(cudaMemcpy(out.data(), dO.p, out.size() * 4, cudaMemcpyDeviceToHost));
  *ok_shifts = 0;
  for (int r = 0; r <= 8; r++) {
    bool ok = true;
    for (int ks = 0; ks < 2; ks++)
      for (int m = 0; m < 64; m++)
        for (int n = 0; n < P::BN; n++) {
          float ref = 0.f;
          for (int k = 0; k < 16; k++)
            ref += Af[(m + (SHIFT_B ? 0 : r)) * 32 + 16 * ks + k] * Bf[(n + (SHIFT_B ? r : 0)) * 32 + 16 * ks + k];
          if (out[((r * 2 + ks) * 64 + m) * P::BN + n] != ref) ok = false;
        }
    if (ok) *ok_shifts |= 1u << r;
  }
  return 0;
}

int selftest_wgmma_row_shift(bool shift_b, int base_offset_mode, unsigned* ok_shifts) {
  return shift_b ? selftest_row_shift<true>(base_offset_mode, ok_shifts) : selftest_row_shift<false>(base_offset_mode, ok_shifts);
}

// ------------------------------------------------------------------------------------ 16-bit hi/lo split
// x [rows_in, ld_in] float32 -> hi/lo 16-bit planes [rows_out, ld_out]; optionally MaxPool1d(3) over rows
// (out row r <- max of in rows 3r..3r+2) and the previous InstanceNorm1d + LeakyReLU (scale/shift per
// (item, channel), item = out row / item_rows); channels [C, ld_out) are written as zeros.
__global__ void __launch_bounds__(256) split_kernel(const float* __restrict__ x, long long rows_out, int C, int ld_in,
                                                    int ld_out, int pool, int item_rows, const float* __restrict__ sc,
                                                    const float* __restrict__ sh, __nv_bfloat16* __restrict__ hi,
                                                    __nv_bfloat16* __restrict__ lo, const int* __restrict__ skip_flag) {
  if (skip_flag && *skip_flag != 0) return;
  const int q_per_row = ld_out >> 2;
  const long long n4 = rows_out * q_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / q_per_row;
    const int c = (int)(i - row * q_per_row) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C) {
      if (pool) {
        const float* p = x + (row * 3) * ld_in + c;
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + ld_in),
                     d = *reinterpret_cast<const float4*>(p + 2 * ld_in);
        v = make_float4(fmaxf(fmaxf(a.x, b.x), d.x), fmaxf(fmaxf(a.y, b.y), d.y), fmaxf(fmaxf(a.z, b.z), d.z),
                        fmaxf(fmaxf(a.w, b.w), d.w));
      } else {
        v = *reinterpret_cast<const float4*>(x + row * ld_in + c);
      }
      if (sc) {
        const long long item = row / item_rows;
        const float4 s = *reinterpret_cast<const float4*>(sc + item * ld_in + c);
        const float4 h = *reinterpret_cast<const float4*>(sh + item * ld_in + c);
        v.x = leaky(fmaf(v.x, s.x, h.x)); v.y = leaky(fmaf(v.y, s.y, h.y));
        v.z = leaky(fmaf(v.z, s.z, h.z)); v.w = leaky(fmaf(v.w, s.w, h.w));
      }
    }
    uint16_t h0, h1, h2, h3, l0, l1, l2, l3;
    split_h16(v.x, h0, l0);
    split_h16(v.y, h1, l1);
    split_h16(v.z, h2, l2);
    split_h16(v.w, h3, l3);
    reinterpret_cast<uint2*>(hi)[i] = make_uint2(pack_u16x2(h0, h1), pack_u16x2(h2, h3));
    reinterpret_cast<uint2*>(lo)[i] = make_uint2(pack_u16x2(l0, l1), pack_u16x2(l2, l3));
  }
}

int launch_split_ex(const float* x, long long rows_out, int C, int ld_in, int ld_out, int pool, int item_rows,
                    const float* sc, const float* sh, void* hi, void* lo, cudaStream_t st, const int* skip_flag) {
  ProfScope _ps("split16", st);
  if (C % 4 || ld_in % 4 || ld_out % 4) {
    set_error("split: channel counts must be multiples of 4");
    return -1;
  }
  const long long n4 = rows_out * (ld_out / 4);
  const long long want = (n4 + 255) / 256;
  const int cap = usable_sms() * 16;
  const int grid = (int)(want < cap ? want : cap);
  split_kernel<<<grid, 256, 0, st>>>(x, rows_out, C, ld_in, ld_out, pool, item_rows, sc, sh,
                                     reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo), skip_flag);
  DG_LAUNCHED();
  return 0;
}

// host-side fp16 conversions, round to nearest even (subnormals kept, finite overflow saturates like cvt.satfinite)
uint16_t host_f32_to_h16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  const uint32_t sign = (u >> 16) & 0x8000u;
  const uint32_t au = u & 0x7FFFFFFFu;
  if (au > 0x7F800000u) return (uint16_t)(sign | 0x7FFFu);                  // NaN
  if (au >= 0x477FF000u) return (uint16_t)(sign | 0x7BFFu);                 // >= 65520 (or inf): largest finite
  if (au < 0x33000001u) return (uint16_t)sign;                              // <= 2^-25: rounds to zero
  const int e = (int)(au >> 23) - 127;                                      // unbiased exponent
  uint32_t mant = (au & 0x7FFFFFu) | 0x800000u;                             // 24-bit significand
  int shift = e >= -14 ? 13 : 13 + (-14 - e);                               // bits dropped
  uint32_t q = mant >> shift;
  const uint32_t rem = mant & ((1u << shift) - 1u), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1u))) q++;
  // normal: q has the implicit bit at position 10 -> exponent field e + 15 (a carry out of rounding propagates by itself)
  const uint32_t bits = e >= -14 ? (uint32_t)((e + 14) << 10) + q : q;
  return (uint16_t)(sign | bits);
}
float host_h16_to_f32(uint16_t h) {
  const uint32_t sign = ((uint32_t)h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 0x3FFu;
  if (e == 0) {
    const float v = (float)m * 5.9604644775390625e-08f;                  // m * 2^-24
    return sign ? -v : v;
  }
  const uint32_t u = e == 31 ? (sign | 0x7F800000u | (m << 13)) : (sign | ((e + 112u) << 23) | (m << 13));
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// host: float32 [N][K] -> zero-padded fp16 hi/lo planes [Npad][K]
void split_weights_host(const float* w, int N, int Npad, int K, uint16_t* hi, uint16_t* lo, float scale) {
  for (size_t i = 0; i < (size_t)Npad * K; i++) hi[i] = lo[i] = 0;
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) {
      const float f = w[(size_t)n * K + k] * scale;          // power of two: exact
      const uint16_t h = host_f32_to_h16(f);
      hi[(size_t)n * K + k] = h;
      lo[(size_t)n * K + k] = host_f32_to_h16(f - host_h16_to_f32(h));
    }
}

// Power-of-two scale of a weight tensor's fp16 planes: the largest magnitude lands in [2^12, 2^13), so that the lo plane
// (|lo| <= 2^-11 |w|) of every weight down to 2^-15 of the largest one stays a NORMAL fp16 number (un-scaled, lo goes
// subnormal below |w| = 0.125 and the pair keeps only an absolute 2^-25).  The accumulator is multiplied by 1 / scale in
// the epilogue (an exact operation).
float weight_plane_scale(const float* w, size_t n) {
  float mx = 0.f;
  for (size_t i = 0; i < n; i++) {
    const float v = fabsf(w[i]);
    if (v > mx && v < 3.0e38f) mx = v;
  }
  if (!(mx > 0.f)) return 1.f;
  int e = 0;
  frexpf(mx, &e);                       // mx = m * 2^e, m in [0.5, 1)
  int k = 13 - e;                       // mx * 2^k in [2^12, 2^13)
  k = k > 40 ? 40 : (k < -40 ? -40 : k);
  return ldexpf(1.f, k);
}

}  // namespace dg

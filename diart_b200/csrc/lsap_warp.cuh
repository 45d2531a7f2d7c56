// Warp-collective rectangular linear sum assignment (scipy.optimize.linear_sum_assignment's algorithm and tie-breaking),
// shared by the clustering (cluster.cu, up to 8 rows) and the DER scoring (der.cu, up to 32 rows).
#pragma once
#include <math.h>

namespace dg {

constexpr unsigned FULL = 0xffffffffu;

// warp-wide minimum of a double through two 32-bit redux.sync steps on an order-preserving integer
// key (10 dependent shuffles otherwise; the assignment logic is a chain of such reductions)
__device__ __forceinline__ double warp_min_d(double v) {
  v += 0.0;   // -0.0 -> +0.0 so that key order == numeric order for equal values
  const long long b = __double_as_longlong(v);
  const unsigned long long key = (unsigned long long)(b ^ ((b >> 63) | (long long)0x8000000000000000ull));
  const unsigned hi = (unsigned)(key >> 32);
  const unsigned mh = __reduce_min_sync(FULL, hi);
  const unsigned ml = __reduce_min_sync(FULL, hi == mh ? (unsigned)key : 0xffffffffu);
  const unsigned long long mk = ((unsigned long long)mh << 32) | ml;
  const long long mb = (long long)(mk ^ (((long long)mk >> 63) ? 0x8000000000000000ull : 0xffffffffffffffffull));
  return __longlong_as_double(mb);
}

// c[i] of a register array without dynamic indexing (which would place the array in local memory)
template <int RK>
__device__ __forceinline__ double sel(const double (&c)[RK], int i) {
  double r = c[0];
#pragma unroll
  for (int q = 1; q < RK; q++) r = (i == q) ? c[q] : r;
  return r;
}

// Column-parallel rectangular LSAP (nr <= nc <= 32, nr <= RK), warp-collective, all state in registers:
// lane j holds column j's dual v, shortest-path cost, predecessor and position in scipy's `remaining`
// list; lane i (i < nr) also holds row i's dual u and its column.  cost[i] is C[i][lane].
// Returns, in lane i < nr, the column assigned to row i.  Arithmetic and tie-breaking follow scipy's
// implementation of Crouse's algorithm: r = ((minVal + c) - u) - v; among equal shortest-path costs
// prefer an unassigned column, scanning `remaining` (initialised in reverse, swap-removed) in order.
template <int RK>
__device__ int lsap_warp(const double (&cost)[RK], int nr, int nc, int lane) {
  double v = 0.0, u = 0.0;
  int row4col = -1, c4r = -1;
  for (int cur = 0; cur < nr; cur++) {
    double minVal = 0.0, spc = INFINITY;
    int i = cur, pos = nc - 1 - lane, path = -1, num = nc, sink = -1;
    bool rem = lane < nc, sc = false;
    unsigned visited = 0;
    while (sink < 0) {
      visited |= 1u << i;
      const double ui = __shfl_sync(FULL, u, i);
      if (rem) {
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, sel(cost, i)), ui), v);
        if (r < spc) {
          path = i;
          spc = r;
        }
      }
      const double lowest = warp_min_d(rem ? spc : INFINITY);
      const bool is_c = rem && spc == lowest;
      const unsigned cand = __ballot_sync(FULL, is_c);
      const unsigned candfree = __ballot_sync(FULL, is_c && row4col < 0);
      if (cand == 0) return c4r;  // infeasible (never: all costs are finite)
      // candfree: the candidate with the largest list position; else the smallest
      const bool mine = candfree ? (is_c && row4col < 0) : is_c;
      const int key = mine ? (candfree ? pos : 64 - pos) : -1;
      const int best = __reduce_max_sync(FULL, key);
      const int j = __ffs(__ballot_sync(FULL, mine && key == best)) - 1;
      minVal = lowest;
      const int r4c = __shfl_sync(FULL, row4col, j);
      const int idx = __shfl_sync(FULL, pos, j);
      if (r4c < 0) sink = j;
      else i = r4c;
      if (lane == j) {
        sc = true;
        rem = false;
      } else if (rem && pos == num - 1) {
        pos = idx;
      }
      num--;
    }
    // dual updates (rows: one per lane; uses the pre-augmentation col4row)
    const double sp = __shfl_sync(FULL, spc, c4r >= 0 ? c4r : 0);
    if (lane == cur) u = __dadd_rn(u, minVal);
    else if (lane < nr && ((visited >> lane) & 1u)) u = __dadd_rn(u, __dsub_rn(minVal, sp));
    if (sc) v = __dsub_rn(v, __dsub_rn(minVal, spc));
    // augment along the path
    int j = sink;
    while (true) {
      const int pi = __shfl_sync(FULL, path, j);
      if (lane == j) row4col = pi;
      const int prev = __shfl_sync(FULL, c4r, pi);
      if (lane == pi) c4r = j;
      j = prev;
      if (pi == cur) break;
    }
  }
  return c4r;
}

}  // namespace dg

// Moving live streams between dg_multi handles (dg_multi_export / dg_multi_import): one kernel copies a list of pieces of
// 32-bit words, each from a linear array or a ring to a linear array or a ring.  Export gathers every listed slot's device
// state into a staging buffer laid out as the packed states; import scatters a staging buffer of packed states into slots.
#include "dg_common.cuh"

namespace dg {

// CTA b takes pieces b, b + gridDim.x, ... (the shape of ring_scatter), its threads the words of each piece.  A ring index is
// reduced once per thread and piece and then moved on by subtraction, so no word costs a 64-bit division.
__global__ void __launch_bounds__(256) slot_transfer_kernel(const XferPiece* __restrict__ pieces, int n_pieces) {
  for (int q = blockIdx.x; q < n_pieces; q += gridDim.x) {
    const XferPiece p = pieces[q];
    long long s = p.src_mod ? (p.src_pos + threadIdx.x) % p.src_mod : p.src_pos + threadIdx.x;
    long long d = p.dst_mod ? (p.dst_pos + threadIdx.x) % p.dst_mod : p.dst_pos + threadIdx.x;
    for (long long i = threadIdx.x; i < p.n; i += blockDim.x) {
      p.dst[d] = __ldg(p.src + s);
      s += blockDim.x;
      d += blockDim.x;
      if (p.src_mod) while (s >= p.src_mod) s -= p.src_mod;
      if (p.dst_mod) while (d >= p.dst_mod) d -= p.dst_mod;
    }
  }
}

int launch_slot_transfer(const XferPiece* pieces, int n_pieces, const char* tag, cudaStream_t st) {
  ProfScope _ps(tag, st);
  if (n_pieces < 1) return 0;
  slot_transfer_kernel<<<n_pieces < 4096 ? n_pieces : 4096, 256, 0, st>>>(pieces, n_pieces);
  DG_LAUNCHED();
  return 0;
}

}  // namespace dg

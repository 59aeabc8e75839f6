// Warp-wide top-32 of (key, index) pairs in ascending lexicographic order, shared by the all-pairs select
// (knn_select.cu) and the cell-grid radius select (radius_select.cu): lane l holds the l-th smallest pair.
#pragma once
#include "common.cuh"

namespace egnn {

template <typename T>
__device__ __forceinline__ bool lex_less(T ka, int ia, T kb, int ib) {
  return ka < kb || (ka == kb && ia < ib);
}

// One compare-exchange step of a warp bitonic network on (key, idx) pairs.
template <typename T>
__device__ __forceinline__ void cmpex(T& key, int& idx, int lane, int partner_xor, bool ascending_block) {
  T ok = shfl_xor_t<T>(key, partner_xor);
  int oi = __shfl_xor_sync(0xffffffffu, idx, partner_xor);
  const bool lower = (lane & partner_xor) == 0;
  const bool other_less = lex_less<T>(ok, oi, key, idx);
  // in an ascending block the lower lane keeps the min
  const bool take_other = (lower == ascending_block) ? other_less : !other_less && !(ok == key && oi == idx);
  if (take_other) { key = ok; idx = oi; }
}

template <typename T>
__device__ __forceinline__ void warp_sort_asc(T& key, int& idx, int lane) {
#pragma unroll
  for (int size = 2; size <= 32; size <<= 1) {
    const bool asc = (lane & size) == 0 || size == 32;
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) cmpex<T>(key, idx, lane, stride, asc);
  }
}

// best (sorted ascending across lanes) <- the 32 smallest of best U cand.
template <typename T>
__device__ __forceinline__ void warp_merge(T& bkey, int& bidx, T ckey, int cidx, int lane) {
  warp_sort_asc<T>(ckey, cidx, lane);
  // reverse the candidates so that best ++ reversed(cand) is bitonic; lane l meets cand[31-l]
  T rk = shfl_idx_t<T>(ckey, 31 - lane);
  int ri = __shfl_sync(0xffffffffu, cidx, 31 - lane);
  if (lex_less<T>(rk, ri, bkey, bidx)) { bkey = rk; bidx = ri; }
  // the kept 32 form a bitonic sequence: finish with the 5 merge steps
#pragma unroll
  for (int stride = 16; stride > 0; stride >>= 1) cmpex<T>(bkey, bidx, lane, stride, true);
}

}  // namespace egnn

// The pieces of the neighbour selects shared by the all-pairs select (knn_select.cu) and the cell-grid selects
// (radius_select.cu): the pair rank, the per-row lattice, the warp-wide top-32 of (key, index) pairs in ascending
// lexicographic order (lane l holds the l-th smallest pair), the k <= 32 warp list built on it, and the bitonic
// network on (key, index) pairs in shared memory with the k > 32 list built on it.
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

// Graph b's lattice as a row ranks under it, staged once per row: its box (bl, binv; box_axis) under PBC_BOX, its cell
// (pc; cell_staged) under PBC_CELL.  NC bounds the coordinate count C.
template <typename T, int NC, int PBC>
struct RowLattice {
  T bl[PBC == PBC_BOX ? NC : 1], binv[PBC == PBC_BOX ? NC : 1];
  T pc[PBC == PBC_CELL ? CELL_STAGED : 1];
  __device__ __forceinline__ RowLattice(const T* box, int b, int C) {
    if constexpr (PBC == PBC_CELL) {
#pragma unroll
      for (int t = 0; t < CELL_STAGED; ++t) pc[t] = cell_staged<T>(box, b, C, t);
    } else if constexpr (PBC) {
#pragma unroll
      for (int c = 0; c < NC; ++c) box_axis<T>(box, b, C, c, bl[c], binv[c]);
    }
  }
};

// The rank of the pair (x_i, x_j): the squared length of x_i - x_j, wrapped by min_image per axis under a box (bl,
// binv) or by cell_wrap under a cell (pc), summed with sq_acc in axis order in the coordinates' type.  xj(c) reads
// coordinate c of x_j.  The loops run to the compile-time NC with a c < C guard, so that C == NC known at compile time
// leaves straight-line code.
template <typename T, int NC, int PBC, class XJ>
__device__ __forceinline__ T pair_rank(const T* xi, XJ xj, int C, const T* bl, const T* binv, const T* pc) {
  T d = T(0);
  if constexpr (PBC == PBC_CELL) {
    T r[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = (c < NC && c < C) ? xi[c < NC ? c : 0] - xj(c < NC ? c : 0) : T(0);
    cell_wrap<T>(r[0], r[1], r[2], pc);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      if (c < NC && c < C) d = sq_acc<T>(r[c], d);
  } else {
#pragma unroll
    for (int c = 0; c < NC; ++c)
      if (c < C) {
        T r = xi[c] - xj(c);
        if constexpr (PBC) r = min_image<T>(r, bl[c], binv[c]);
        d = sq_acc<T>(r, d);
      }
  }
  return d;
}

// The all-pairs select's rank of (i, j) from its pair_rank d (reference egnn_pytorch.py:240-256): 1e5 when the pair is
// masked (a mask is given and either end is padded); under an adjacency row, -1 for i == j and 0 for an adjacent j.
template <typename T>
__device__ __forceinline__ T select_rank(T d, bool masked, const uint8_t* adjrow, int i, int j) {
  if (masked) d = T(1e5);
  if (adjrow) {
    if (i == j) d = T(-1);
    else if (adjrow[j]) d = T(0);
  }
  return d;
}

// k <= 32: lane l keeps the l-th smallest (rank, j) so far (bkey, bidx); pairs that beat the k-th are queued in the
// warp's 64 queue slots (qk, qi) and merged 32 at a time (warp_merge).
template <typename T>
struct LaneList {
  T* qk;
  int* qi;
  int k;
  T bkey = T(INFINITY), thr_key = T(INFINITY);   // lane l: l-th smallest so far; the k-th smallest so far
  int bidx = 0x7fffffff, thr_idx = 0x7fffffff;
  int count = 0;                                 // queued pairs (warp-uniform)
  __device__ __forceinline__ LaneList(T* qk_, int* qi_, int k_) : qk(qk_), qi(qi_), k(k_) {}
  __device__ __forceinline__ bool beats(T key, int j) const { return lex_less<T>(key, j, thr_key, thr_idx); }
  // queues the pairs of the lanes whose `pass` is set; called by the whole warp
  __device__ __forceinline__ void push(bool pass, T key, int j, int lane) {
    const unsigned bal = __ballot_sync(0xffffffffu, pass);
    if (bal == 0) return;
    if (pass) {
      const int q = count + __popc(bal & ((1u << lane) - 1));
      qk[q] = key;
      qi[q] = j;
    }
    count += __popc(bal);
    __syncwarp();
    if (count >= 32) {
      T ckey = qk[lane];
      int cidx = qi[lane];
      __syncwarp();
      if (lane + 32 < count) {         // shift the tail of the queue down
        T tk = qk[lane + 32]; int ti = qi[lane + 32];
        qk[lane] = tk; qi[lane] = ti;
      }
      count -= 32;
      __syncwarp();
      warp_merge<T>(bkey, bidx, ckey, cidx, lane);
      refresh();
    }
  }
  // merges what is still queued: lane l then holds the l-th smallest of every pair pushed
  __device__ __forceinline__ void finish(int lane) {
    if (count > 0) {
      T ckey = lane < count ? qk[lane] : T(INFINITY);
      int cidx = lane < count ? qi[lane] : 0x7fffffff;
      warp_merge<T>(bkey, bidx, ckey, cidx, lane);
      count = 0;
    }
  }
  __device__ __forceinline__ void refresh() {
    thr_key = shfl_idx_t<T>(bkey, k - 1);
    thr_idx = __shfl_sync(0xffffffffu, bidx, k - 1);
  }
};

// Steps stride = half, half/2, .., 1 of the bitonic network on n = 2^m (key, idx) pairs in shared memory, each run by
// the threads tid = 0 .. nthreads-1 and followed by sync(): the pair (lo, hi = lo + stride) is put in ascending
// (lexicographic) order where lo & dir == 0, in descending order elsewhere.
template <typename T, class Sync>
__device__ __forceinline__ void bitonic_steps(T* key, int* idx, int n, int half, int dir, int tid, int nthreads,
                                              Sync sync) {
  for (int stride = half; stride > 0; stride >>= 1) {
    for (int t = tid; t < n / 2; t += nthreads) {
      const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;    // index with the `stride` bit clear
      const bool asc = (lo & dir) == 0;
      if (lex_less<T>(key[hi], idx[hi], key[lo], idx[lo]) == asc) {
        const T tk = key[lo]; key[lo] = key[hi]; key[hi] = tk;
        const int ti = idx[lo]; idx[lo] = idx[hi]; idx[hi] = ti;
      }
    }
    sync();
  }
}

// Sorts n = 2^m (key, idx) pairs in shared memory ascending: merges bitonic blocks of size = 2, 4, .., n, each block
// ascending where its index has the `size` bit clear.
template <typename T, class Sync>
__device__ __forceinline__ void bitonic_sort(T* key, int* idx, int n, int tid, int nthreads, Sync sync) {
  for (int size = 2; size <= n; size <<= 1) bitonic_steps<T>(key, idx, n, size >> 1, size, tid, nthreads, sync);
}

// Sorts a bitonic sequence of n = 2^m (key, idx) pairs in shared memory ascending.
template <typename T, class Sync>
__device__ __forceinline__ void bitonic_merge(T* key, int* idx, int n, int tid, int nthreads, Sync sync) {
  bitonic_steps<T>(key, idx, n, n >> 1, 0, tid, nthreads, sync);
}

// k > 32: the top k kept in shared memory instead of lanes.  Per warp, KP = next_pow2(k) (>= 64) pairs
// `list` (lk, li), sorted ascending (the KP smallest (rank, j) so far, padded with (inf, IMAX)), and KP more `queue`.  A
// pair that beats the current k-th list entry is queued.  Once the queue could not take another 32, it is padded,
// sorted and merged into the list: list[s] = min(list[s], queue[KP-1-s]) leaves the KP smallest of both as a bitonic
// sequence, which log2(KP) merge steps sort.  The list is a function of the set of pairs queued, and every pair the
// filter drops is beaten by k listed ones, so the k kept pairs are the k smallest of all pairs offered, whatever order
// they arrive in.
template <typename T>
struct SmemList {
  T* lk;
  int* li;
  T* qk;
  int* qi;
  int KP, k;
  T thr_key = T(INFINITY);             // the k-th smallest so far
  int thr_idx = 0x7fffffff;
  int count = 0;                       // queued pairs (warp-uniform)
  __device__ __forceinline__ SmemList(T* lk_, int* li_, int KP_, int k_, int lane)
      : lk(lk_), li(li_), qk(lk_ + KP_), qi(li_ + KP_), KP(KP_), k(k_) {
    for (int s = lane; s < KP; s += 32) { lk[s] = T(INFINITY); li[s] = 0x7fffffff; }
  }
  __device__ __forceinline__ bool beats(T key, int j) const { return lex_less<T>(key, j, thr_key, thr_idx); }
  __device__ __forceinline__ void flush(int lane) {
    for (int s = count + lane; s < KP; s += 32) { qk[s] = T(INFINITY); qi[s] = 0x7fffffff; }
    __syncwarp();
    bitonic_sort<T>(qk, qi, KP, lane, 32, [] { __syncwarp(); });
    for (int s = lane; s < KP; s += 32) {
      const T ck = qk[KP - 1 - s];
      const int ci = qi[KP - 1 - s];
      if (lex_less<T>(ck, ci, lk[s], li[s])) { lk[s] = ck; li[s] = ci; }
    }
    __syncwarp();
    bitonic_merge<T>(lk, li, KP, lane, 32, [] { __syncwarp(); });
    count = 0;
    thr_key = lk[k - 1];
    thr_idx = li[k - 1];
  }
  // queues the pairs of the lanes whose `pass` is set; called by the whole warp
  __device__ __forceinline__ void push(bool pass, T key, int j, int lane) {
    const unsigned bal = __ballot_sync(0xffffffffu, pass);
    if (bal == 0) return;
    if (pass) {
      const int q = count + __popc(bal & ((1u << lane) - 1));
      qk[q] = key;
      qi[q] = j;
    }
    count += __popc(bal);
    if (count > KP - 32) flush(lane);
  }
  __device__ __forceinline__ void finish(int lane) {
    if (count > 0) flush(lane);
  }
  __device__ __forceinline__ void refresh() {
    __syncwarp();
    thr_key = lk[k - 1];
    thr_idx = li[k - 1];
  }
};

// Dynamic shared memory of a SmemList warp, and its list length for k: next_pow2(k), at least 64.
inline size_t smem_list_bytes(int KP, size_t tbytes) { return (size_t)2 * KP * (tbytes + sizeof(int)); }
inline int list_kp(int k) {
  int KP = 64;
  while (KP < k) KP <<= 1;
  return KP;
}

}  // namespace egnn

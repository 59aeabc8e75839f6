// Segmented neighbour select: k-nearest lists for a packed batch of variable-size graphs.  The batch is one node axis
// of T nodes cut into G contiguous segments by int32 offsets ptr[G+1] (graph g = nodes [ptr[g], ptr[g+1]), PyTorch
// Geometric's `ptr`), and every node is ranked against the nodes of its own segment only: O(sum_g n_g^2) pair ranks
// instead of the O(G N_max^2) of the same batch padded to [G, N_max].
//
// A node's list equals egnn_knn_select's for its segment alone (B = 1, N = n_g) bit for bit, with indices into the
// node axis: the same rank (pair_rank, select_rank: 1e5 to and from a padded node), the same (rank, j) lexicographic
// order -- segments are contiguous, so global indices order as local ones -- and the same NaN-last rule.  A NaN rank is
// offered as (+inf, j + T), after every finite or +inf rank and in index order, and written as j with ok = 0, as
// knn_block_sort_kernel does.  Slots past n_g (n_g < k) are written as -1 with ok = 0.
//
// Two launches, neither synchronising with the host (so the call can be captured in a CUDA graph):
//   tiles   one CTA: the exclusive prefix of each segment's row tiles, ceil(n_g / SEG_WARPS), into the workspace
//   select  one CTA per tile, launched for the bound ceil(T / SEG_WARPS) + G of the tile count (surplus CTAs exit):
//           SEG_WARPS rows of one segment, one warp each, stage the segment's candidates in shared-memory chunks of
//           SEG_JC (coordinates as SoA and mask bytes), rank them and keep the top k in a LaneList (k <= 32) or a
//           SmemList (k > 32).
// Segment bounds are clamped to [0, T] on the device, so no ptr can make a kernel read or write out of range.
//
// The grid entries (egnn_radius_select_packed, egnn_knn_grid_select_packed) put every graph of at least the unpacked
// threshold's nodes (and at least k) on the radius or kNN grid of radius_select.cu in its segment form, and the rest on
// this select: seg_grid_tiles_kernel gives the grid graphs 0 row tiles and checks ptr (non-decreasing within [0, T]:
// the graphs' node ranges and bucket regions are then disjoint; any other ptr puts every graph on this select), the
// grid's launches follow, then the select.  A call whose largest graph is below the threshold issues the two launches
// above and nothing else.
#include "common.cuh"
#include "profile.h"
#include "warp_select.cuh"
#include <cub/block/block_scan.cuh>

namespace egnn {

constexpr int SEG_WARPS = 8;            // rows per CTA, all of one segment
constexpr int SEG_JC = 1024;            // candidates staged per pass
constexpr int SEG_TILE_THREADS = 1024;  // the tile scan: one CTA
constexpr int SEG_MAX_K = 256;
constexpr int SEG_MAX_T = 1 << 30;      // j + T, the index of a NaN rank, stays an int

template <typename T>
struct SegArgs {
  int G, T_, C, k;
  const int32_t* ptr;     // [G+1]
  const T* coors;         // [T, C]
  const uint8_t* mask;    // [T] or null
  const T* box;           // [C] box (PBC_BOX) or [C, C] cell (PBC_CELL), shared by every segment
  T valid_radius;
  int32_t* out_idx;       // [T, k]
  uint8_t* out_ok;        // [T, k] or null
  const int* tile0;       // [G+1] first tile of each segment; tile0[G] = the tile count
  int KP;                 // SmemList length (k > 32)
};

__device__ __forceinline__ void seg_bounds(const int32_t* ptr, int g, int T, int& lo, int& hi) {
  lo = min(max(ptr[g], 0), T);
  hi = min(max(ptr[g + 1], lo), T);
}

__global__ void __launch_bounds__(SEG_TILE_THREADS) seg_tiles_kernel(const int32_t* __restrict__ ptr, int G, int T,
                                                                     int* __restrict__ tile0) {
  using Scan = cub::BlockScan<int, SEG_TILE_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int g0 = 0; g0 < G; g0 += SEG_TILE_THREADS) {
    const int g = g0 + threadIdx.x;
    int tiles = 0;
    if (g < G) {
      int lo, hi;
      seg_bounds(ptr, g, T, lo, hi);
      tiles = ceil_div(hi - lo, SEG_WARPS);
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(tiles, excl, total);
    if (g < G) tile0[g] = carry + excl;
    carry += total;
    __syncthreads();                    // tmp is reused by the next chunk
  }
  if (threadIdx.x == 0) tile0[G] = carry;
}

// seg_tiles_kernel beside a grid: 0 tiles for each graph of at least min_n nodes when ptr is valid, whose validity goes
// to *valid for the grid's kernels.
__global__ void __launch_bounds__(SEG_TILE_THREADS) seg_grid_tiles_kernel(const int32_t* __restrict__ ptr, int G, int T,
                                                                          int min_n, int* __restrict__ tile0,
                                                                          int* __restrict__ valid) {
  using Scan = cub::BlockScan<int, SEG_TILE_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  int bad = 0;
  for (int g = threadIdx.x; g <= G; g += SEG_TILE_THREADS) {
    const int v = ptr[g];
    bad |= v < 0 || v > T || (g < G && ptr[g + 1] < v);
  }
  const bool ok = !__syncthreads_or(bad);
  int carry = 0;
  for (int g0 = 0; g0 < G; g0 += SEG_TILE_THREADS) {
    const int g = g0 + threadIdx.x;
    int tiles = 0;
    if (g < G) {
      int lo, hi;
      seg_bounds(ptr, g, T, lo, hi);
      tiles = ok && hi - lo >= min_n ? 0 : ceil_div(hi - lo, SEG_WARPS);
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(tiles, excl, total);
    if (g < G) tile0[g] = carry + excl;
    carry += total;
    __syncthreads();                    // tmp is reused by the next chunk
  }
  if (threadIdx.x == 0) { tile0[G] = carry; *valid = ok ? 1 : 0; }
}

// Shared memory of the select: staged coordinates [C][SEG_JC], the lists of SEG_WARPS warps, mask bytes [SEG_JC].
template <typename T>
inline size_t seg_smem_bytes(int C, int k) {
  const size_t lists = k > 32 ? SEG_WARPS * smem_list_bytes(list_kp(k), sizeof(T))
                              : (size_t)SEG_WARPS * 64 * (sizeof(T) + sizeof(int));
  return (size_t)C * SEG_JC * sizeof(T) + lists + SEG_JC;
}

// CDIM = 3: straight-line coordinate loops (the generic instantiation, CDIM = 0, runs to 8 with a c < C guard).
template <typename T, int CDIM, int PBC, bool WIDE>
__global__ void __launch_bounds__(SEG_WARPS * 32) seg_select_kernel(const SegArgs<T> a) {
  constexpr int NC = CDIM ? CDIM : 8;
  extern __shared__ __align__(16) unsigned char seg_sm[];
  const int tile = blockIdx.x;
  if (tile >= a.tile0[a.G]) return;     // surplus CTA of the launch bound (CTA-uniform)
  int glo = 0, ghi = a.G - 1;           // the segment g owning the tile: the last g with tile0[g] <= tile
  while (glo < ghi) {
    const int mid = (glo + ghi + 1) >> 1;
    if (a.tile0[mid] <= tile) glo = mid; else ghi = mid - 1;
  }
  int lo, hi;
  seg_bounds(a.ptr, glo, a.T_, lo, hi);
  const int n = hi - lo;
  const int C = CDIM ? CDIM : a.C;
  T* xs = reinterpret_cast<T*>(seg_sm);                                   // [C][JC]
  unsigned char* lists = seg_sm + (size_t)C * SEG_JC * sizeof(T);
  const size_t list_bytes = (size_t)SEG_WARPS * (WIDE ? 2 * a.KP : 64) * (sizeof(T) + sizeof(int));   // seg_smem_bytes
  uint8_t* ms = lists + list_bytes;                                       // [JC]
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int iraw = lo + (tile - a.tile0[glo]) * SEG_WARPS + warp;
  const bool rv = iraw < hi;
  const int i = rv ? iraw : hi - 1;     // n >= 1: the segment owns a tile
  T xi[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) xi[c] = (CDIM || c < a.C) ? a.coors[(size_t)i * a.C + c] : T(0);
  const bool mask_i = a.mask ? a.mask[i] != 0 : true;
  const RowLattice<T, NC, PBC> lat(a.box, 0, a.C);
  const int NANOFF = a.T_;

  auto scan = [&](auto& L) {
    for (int jc0 = 0; jc0 < n; jc0 += SEG_JC) {
      const int jn = min(SEG_JC, n - jc0);
      __syncthreads();                  // previous pass fully consumed
      for (int jj = threadIdx.x; jj < jn; jj += SEG_WARPS * 32) {
        const T* src = a.coors + (size_t)(lo + jc0 + jj) * a.C;
#pragma unroll
        for (int c = 0; c < NC; ++c)
          if (CDIM || c < a.C) xs[c * SEG_JC + jj] = src[c];
        if (a.mask) ms[jj] = a.mask[lo + jc0 + jj];
      }
      __syncthreads();
      for (int j0 = 0; j0 < jn; j0 += 32) {
        const int jj = j0 + lane, j = lo + jc0 + jj;
        T key = T(INFINITY);
        int jk = 0x7fffffff;
        bool pass = false;
        if (jj < jn) {
          key = select_rank<T>(pair_rank<T, NC, PBC>(xi, [&](int c) { return xs[c * SEG_JC + jj]; }, C, lat.bl, lat.binv,
                                                      lat.pc),
                               a.mask && !(mask_i && ms[jj]), nullptr, i, j);
          jk = j;
          if (key != key) { key = T(INFINITY); jk = j + NANOFF; }   // NaN rank: after every +inf, by index
          pass = L.beats(key, jk);
        }
        L.push(pass, key, jk, lane);
      }
    }
    L.finish(lane);
  };
  auto put = [&](int s, T key, int jk) {
    if (!rv || s >= a.k) return;
    const size_t o = (size_t)i * a.k + s;
    const bool empty = jk == 0x7fffffff, nan_rank = !empty && jk >= NANOFF;
    a.out_idx[o] = empty ? -1 : (nan_rank ? jk - NANOFF : jk);
    if (a.out_ok) a.out_ok[o] = !empty && !nan_rank && key <= a.valid_radius ? 1 : 0;
  };
  if constexpr (WIDE) {
    T* lk = reinterpret_cast<T*>(lists) + (size_t)warp * 2 * a.KP;
    int* li = reinterpret_cast<int*>(reinterpret_cast<T*>(lists) + (size_t)SEG_WARPS * 2 * a.KP) + (size_t)warp * 2 * a.KP;
    SmemList<T> L(lk, li, a.KP, a.k, lane);
    scan(L);
    __syncwarp();
    for (int s = lane; s < a.k; s += 32) put(s, lk[s], li[s]);
  } else {
    T* qk = reinterpret_cast<T*>(lists) + warp * 64;
    int* qi = reinterpret_cast<int*>(reinterpret_cast<T*>(lists) + SEG_WARPS * 64) + warp * 64;
    LaneList<T> L(qk, qi, a.k);
    scan(L);
    put(lane, L.bkey, L.bidx);
  }
}

template <typename T, int CDIM, int PBC>
static int launch_seg(const SegArgs<T>& a, cudaStream_t st) {
  const bool wide = a.k > 32;
  const size_t smem = seg_smem_bytes<T>(a.C, a.k);
  const unsigned grid = (unsigned)(ceil_div(a.T_, SEG_WARPS) + a.G);
  static bool attr_set[64] = {false};   // once per device: the most either kernel asks for (C = 8 or 3, k = 256)
  int dev = 0;
  EGNN_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 64 && !attr_set[dev]) {
    const int most = (int)seg_smem_bytes<T>(CDIM ? CDIM : 8, SEG_MAX_K);
    EGNN_CUDA_TRY(cudaFuncSetAttribute(seg_select_kernel<T, CDIM, PBC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       most));
    EGNN_CUDA_TRY(cudaFuncSetAttribute(seg_select_kernel<T, CDIM, PBC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       most));
    attr_set[dev] = true;
  }
  if (wide) seg_select_kernel<T, CDIM, PBC, true><<<grid, SEG_WARPS * 32, smem, st>>>(a);
  else seg_select_kernel<T, CDIM, PBC, false><<<grid, SEG_WARPS * 32, smem, st>>>(a);
  EGNN_LAUNCH_CHECK();
  return EGNN_OK;
}

template <typename T, int PBC>
static int launch_seg_c(const SegArgs<T>& a, cudaStream_t st) {
  return a.C == 3 ? launch_seg<T, 3, PBC>(a, st) : launch_seg<T, 0, PBC>(a, st);
}

static size_t seg_ws_bytes(int G) { return round_up((size_t)(G + 1) * sizeof(int), 256); }

static int seg_check(int G, int T, int C, int k, int pbc) {
  if (G < 1 || T < 1 || T > SEG_MAX_T || C < 1 || C > 8 || k < 1) return EGNN_ERR_SHAPE;
  if ((long long)ceil_div(T, SEG_WARPS) + G > 0x7fffffffLL) return EGNN_ERR_SHAPE;
  if (pbc == PBC_CELL && (C < 2 || C > 3)) return EGNN_ERR_SHAPE;
  if (k > SEG_MAX_K) return EGNN_ERR_UNSUPPORTED;
  return EGNN_OK;
}

// tiles_done: tile0 (ws) was written by seg_grid_tiles_kernel, so only the select is launched.
template <typename T>
static int seg_select(int G, int Tn, int C, int k, const int32_t* ptr, const void* coors, const uint8_t* mask,
                      const void* lattice, int pbc, double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* ws,
                      cudaStream_t st, bool tiles_done = false) {
  SegArgs<T> a;
  a.G = G; a.T_ = Tn; a.C = C; a.k = k;
  a.ptr = ptr;
  a.coors = static_cast<const T*>(coors);
  a.mask = mask;
  a.box = static_cast<const T*>(lattice);
  a.valid_radius = (T)valid_radius;
  a.out_idx = out_idx; a.out_ok = out_ok;
  a.tile0 = static_cast<const int*>(ws);
  a.KP = k > 32 ? list_kp(k) : 0;
  if (tiles_done) {
    count_launch(1);
  } else {
    seg_tiles_kernel<<<1, SEG_TILE_THREADS, 0, st>>>(ptr, G, Tn, static_cast<int*>(ws));
    EGNN_LAUNCH_CHECK();
    count_launch(2);
  }
  if (!lattice) return launch_seg_c<T, PBC_NONE>(a, st);
  if (pbc == PBC_CELL) return launch_seg_c<T, PBC_CELL>(a, st);
  return launch_seg_c<T, PBC_BOX>(a, st);
}

static int seg_entry(int pbc, int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, const int32_t* ptr,
                     const void* coors, const uint8_t* mask, const void* lattice, double valid_radius, int32_t* out_idx,
                     uint8_t* out_ok, void* workspace, size_t workspace_bytes, void* stream) {
  if (!ptr || !coors || !out_idx || !workspace || (pbc == PBC_CELL && !lattice)) return EGNN_ERR_NULL;
  EGNN_TRY(seg_check(G, T, C, k, pbc));
  if (dtype != EGNN_DTYPE_F32 && dtype != EGNN_DTYPE_F64) return EGNN_ERR_UNSUPPORTED;
  if ((uintptr_t)workspace & 0xFF) return EGNN_ERR_ALIGN;
  if (workspace_bytes < seg_ws_bytes(G)) return EGNN_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == EGNN_DTYPE_F64)
    return seg_select<double>(G, T, C, k, ptr, coors, mask, lattice, pbc, valid_radius, out_idx, out_ok, workspace, st);
  return seg_select<float>(G, T, C, k, ptr, coors, mask, lattice, pbc, valid_radius, out_idx, out_ok, workspace, st);
}

// ---------------------------------------------------------------- the grid entries

// Scratch: tile0 [G+1] and the validity flag, then the grid's (packed_grid_ws_bytes).
static size_t seg_grid_head_bytes(int G) { return round_up((size_t)(G + 2) * sizeof(int), 256); }

static int seg_grid_check(int G, int T, int C, int k, int pbc) {
  EGNN_TRY(seg_check(G, T, C, k, pbc));
  if (4LL * T > 0x7fffffffLL) return EGNN_ERR_SHAPE;   // int bucket offsets 4 ptr[g]
  return EGNN_OK;
}

static size_t seg_grid_ws_bytes(bool knn, int G, int T, int C) {
  return seg_grid_head_bytes(G) + (C <= 3 ? packed_grid_ws_bytes(knn, G, T, C) : 0);
}

static int seg_grid_entry(bool knn, int pbc, int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                          const int32_t* ptr, const void* coors, const uint8_t* mask, const void* lattice,
                          double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if (!ptr || !coors || !out_idx || !workspace || (pbc == PBC_CELL && !lattice) || (!knn && !out_ok))
    return EGNN_ERR_NULL;
  EGNN_TRY(seg_grid_check(G, T, C, k, pbc));
  if (dtype != EGNN_DTYPE_F32 && dtype != EGNN_DTYPE_F64) return EGNN_ERR_UNSUPPORTED;
  if ((uintptr_t)workspace & 0xFF) return EGNN_ERR_ALIGN;
  if (workspace_bytes < seg_grid_ws_bytes(knn, G, T, C)) return EGNN_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool f64 = dtype == EGNN_DTYPE_F64;
  const int min_n = C <= 3 ? packed_grid_min_n(knn, dtype, k, valid_radius) : INT_MAX;
  if (max_n < min_n)                                 // no graph is large enough: the segmented select alone
    return f64 ? seg_select<double>(G, T, C, k, ptr, coors, mask, lattice, pbc, valid_radius, out_idx, out_ok, workspace, st)
               : seg_select<float>(G, T, C, k, ptr, coors, mask, lattice, pbc, valid_radius, out_idx, out_ok, workspace, st);
  int* tile0 = static_cast<int*>(workspace);
  seg_grid_tiles_kernel<<<1, SEG_TILE_THREADS, 0, st>>>(ptr, G, T, min_n, tile0, tile0 + G + 1);
  EGNN_LAUNCH_CHECK();
  count_launch(1);
  EGNN_TRY(packed_grid_launch(knn, dtype, G, T, C, k, min_n, ptr, tile0 + G + 1, coors, mask, lattice, pbc, valid_radius,
                              out_idx, out_ok, static_cast<char*>(workspace) + seg_grid_head_bytes(G), st));
  return f64 ? seg_select<double>(G, T, C, k, ptr, coors, mask, lattice, pbc, valid_radius, out_idx, out_ok, workspace, st,
                                  true)
             : seg_select<float>(G, T, C, k, ptr, coors, mask, lattice, pbc, valid_radius, out_idx, out_ok, workspace, st,
                                 true);
}

static int seg_grid_ws_entry(bool knn, int32_t G, int32_t T, int32_t C, int32_t k, size_t* out_bytes) {
  if (!out_bytes) return EGNN_ERR_NULL;
  EGNN_TRY(seg_grid_check(G, T, C, k, PBC_NONE));
  *out_bytes = seg_grid_ws_bytes(knn, G, T, C);
  return EGNN_OK;
}

}  // namespace egnn

extern "C" int egnn_knn_select_packed_workspace_bytes(int32_t G, int32_t T, int32_t C, int32_t k, size_t* out_bytes) {
  if (!out_bytes) return EGNN_ERR_NULL;
  EGNN_TRY(egnn::seg_check(G, T, C, k, egnn::PBC_NONE));
  *out_bytes = egnn::seg_ws_bytes(G);
  return EGNN_OK;
}

extern "C" int egnn_knn_select_packed(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, const int32_t* ptr,
                                      const void* coors, const uint8_t* mask, const void* box, double valid_radius,
                                      int32_t* out_idx, uint8_t* out_ok, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  return egnn::seg_entry(egnn::PBC_BOX, dtype, G, T, C, k, ptr, coors, mask, box, valid_radius, out_idx, out_ok,
                         workspace, workspace_bytes, stream);
}

extern "C" int egnn_knn_select_packed_triclinic(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k,
                                                const int32_t* ptr, const void* coors, const uint8_t* mask,
                                                const void* cell, double valid_radius, int32_t* out_idx,
                                                uint8_t* out_ok, void* workspace, size_t workspace_bytes,
                                                void* stream) {
  return egnn::seg_entry(egnn::PBC_CELL, dtype, G, T, C, k, ptr, coors, mask, cell, valid_radius, out_idx, out_ok,
                         workspace, workspace_bytes, stream);
}

extern "C" int egnn_radius_select_packed_workspace_bytes(int32_t G, int32_t T, int32_t C, int32_t k, size_t* out_bytes) {
  return egnn::seg_grid_ws_entry(false, G, T, C, k, out_bytes);
}

extern "C" int egnn_radius_select_packed(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                                         const int32_t* ptr, const void* coors, const uint8_t* mask, const void* box,
                                         double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  return egnn::seg_grid_entry(false, egnn::PBC_BOX, dtype, G, T, C, k, max_n, ptr, coors, mask, box, valid_radius,
                              out_idx, out_ok, workspace, workspace_bytes, stream);
}

extern "C" int egnn_radius_select_packed_triclinic(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k,
                                                   int32_t max_n, const int32_t* ptr, const void* coors,
                                                   const uint8_t* mask, const void* cell, double valid_radius,
                                                   int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                                   size_t workspace_bytes, void* stream) {
  return egnn::seg_grid_entry(false, egnn::PBC_CELL, dtype, G, T, C, k, max_n, ptr, coors, mask, cell, valid_radius,
                              out_idx, out_ok, workspace, workspace_bytes, stream);
}

extern "C" int egnn_knn_grid_select_packed_workspace_bytes(int32_t G, int32_t T, int32_t C, int32_t k,
                                                           size_t* out_bytes) {
  return egnn::seg_grid_ws_entry(true, G, T, C, k, out_bytes);
}

extern "C" int egnn_knn_grid_select_packed(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                                           const int32_t* ptr, const void* coors, const uint8_t* mask, const void* box,
                                           double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  return egnn::seg_grid_entry(true, egnn::PBC_BOX, dtype, G, T, C, k, max_n, ptr, coors, mask, box, valid_radius,
                              out_idx, out_ok, workspace, workspace_bytes, stream);
}

extern "C" int egnn_knn_grid_select_packed_triclinic(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k,
                                                     int32_t max_n, const int32_t* ptr, const void* coors,
                                                     const uint8_t* mask, const void* cell, double valid_radius,
                                                     int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                                     size_t workspace_bytes, void* stream) {
  return egnn::seg_grid_entry(true, egnn::PBC_CELL, dtype, G, T, C, k, max_n, ptr, coors, mask, cell, valid_radius,
                              out_idx, out_ok, workspace, workspace_bytes, stream);
}

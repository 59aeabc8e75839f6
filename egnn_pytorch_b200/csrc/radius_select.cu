// Radius neighbour search on a hashed uniform cell grid: the k nearest nodes within squared distance r2 of every node,
// in O(N * neighbourhood) instead of the all-pairs select's O(N^2) (reference egnn_pytorch.py:237-260 with a mask and
// a finite valid_radius, :296).
//
// The kept slots equal the all-pairs select's (knn_select.cu) ok = 1 slots exactly: the same rank (x_i - x_j per axis,
// min_image under a box, sq_acc in axis order, in the coordinates' type), the same (rank, j) lexicographic order and
// the same warp merge (warp_select.cuh), restricted to rank <= r2.  Padded nodes and nodes with a non-finite coordinate
// are never inserted into the grid, so they are never kept, and their own rows stay empty.
//
// Grid, per graph: cell edge cs = sqrt(r2) (1 + 2^-10).  A periodic axis (finite L > 0) has n = max(1, floor(L / cs))
// cells of width L / n >= cs, positions wrapped into [0, L); an aperiodic axis uses floor(x / cs), clamped to +-2^30.
// A triclinic cell bins its periodic axes in fractional coordinates instead (frac_cells).
// Binning runs in double.  Cell coordinates hash into Tb = next_pow2(2N) buckets, so the scratch follows from N alone;
// a collision only adds candidates that the exact rank filter removes.  DESIGN.md section 5 gives the argument that
// no pair the filter keeps lies outside the 3^C cells around a node.
//
// Four launches (after one memset of the bucket counts), none synchronising with the host:
//   count   bucket sizes (atomics); non-insertable nodes write their empty rows
//   scan    exclusive prefix of the bucket sizes, one CTA per graph
//   scatter coordinates (SoA) and node indices into cell order; afterwards end[t] is the end of bucket t
//   query   one warp per node, nodes taken in cell order: the deduplicated buckets of the 3^C cells around the node
//           are read as one flattened candidate stream, filtered by rank <= r2 and against the current k-th entry,
//           queued and merged 32 at a time; for k > 32 (radius_query_wide_kernel) the list lives in shared memory.
#include "common.cuh"
#include "profile.h"
#include "warp_select.cuh"
#include <cub/block/block_scan.cuh>

namespace egnn {

constexpr int RS_THREADS = 256;          // count / scatter
constexpr int RS_SCAN_THREADS = 1024;    // scan: one CTA per graph, 4 buckets per thread per tile
constexpr int RS_WARPS = 8;              // query rows per CTA
constexpr int RS_WIDE_MAX_K = 256;       // the longest list the query keeps (radius_query_wide_kernel above 32)
constexpr size_t RS_WIDE_SMEM = 32768;   // wide query: dynamic shared memory per CTA, within the 48 KiB default
constexpr double RS_CLAMP = 1073741824.0;     // 2^30: aperiodic cell coordinates and periodic cell counts

// Buckets per graph: next_pow2(2N).
static inline int rs_buckets(int N) {
  int t = 2;
  while (t < 2 * N) t <<= 1;
  return t;
}

struct CellWs { size_t cnt, end, xs, idx, total; };
static CellWs cell_ws_layout(int B, int N, int C, size_t coord_bytes) {
  CellWs w;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += round_up(bytes, 256); return r; };
  const size_t nb = (size_t)B * rs_buckets(N), nodes = (size_t)B * N;
  w.cnt = take(nb * sizeof(int));
  w.end = take(nb * sizeof(int));
  w.xs = take((size_t)C * nodes * coord_bytes);
  w.idx = take(nodes * sizeof(int));
  w.total = o;
  return w;
}

size_t cell_select_ws_bytes(int B, int N, int C, size_t coord_bytes) { return cell_ws_layout(B, N, C, coord_bytes).total; }

bool cell_select_eligible(const EgnnLayerDesc& d) {
  const int max_k = (d.flags & EGNN_FLAG_CELL_SELECT_WIDE) ? RS_WIDE_MAX_K : 32;
  if (d.k < 1 || d.k > max_k || d.C < 1 || d.C > 3) return false;
  if (d.flags & (EGNN_FLAG_ONLY_SPARSE | EGNN_FLAG_ADJ_BATCHED | EGNN_FLAG_EDGES_PER_SLOT)) return false;
  // the radius in the coordinates' type, as the select compares it; at or above 1e5 padded pairs (rank 1e5) could
  // take slots in the reference
  const double r2 = d.dtype == EGNN_DTYPE_F64 ? d.valid_radius : (double)(float)d.valid_radius;
  return r2 > 0.0 && r2 < 1e5;
}

size_t cell_select_layer_ws_bytes(const EgnnLayerDesc& d) {
  return cell_select_eligible(d) ? cell_select_ws_bytes(d.B, d.N, d.C, d.dtype == EGNN_DTYPE_F64 ? 8 : 4) : 0;
}

// Smallest N per graph at which an eligible layer runs the cell grid (DESIGN.md section 6).  EGNN_B200_CELL_SELECT_MIN_N
// overrides it (0 = always, a huge value = never); read at every call, so one process can run and time both paths.
constexpr long CELL_SELECT_MIN_N = 4096;
static long cell_select_min_n() {
  const char* e = getenv("EGNN_B200_CELL_SELECT_MIN_N");
  return e ? strtol(e, nullptr, 10) : CELL_SELECT_MIN_N;
}

bool cell_select_runs(const EgnnLayerDesc& d, const EgnnLayerIO& io) {
  return io.mask && !io.adj && !io.nbr_idx && cell_select_eligible(d) && d.N >= cell_select_min_n();
}

template <typename T>
struct RadArgs {
  int B, N, k, Tb;
  T r2;
  double cs;                       // cell edge
  const T* coors;                  // [B,N,C]
  const uint8_t* mask;             // [B,N] or null
  const T* box;                    // [B,C] box (PBC_BOX) or [B,C,C] cell (PBC_CELL)
  int* cnt;                        // [B,Tb] bucket sizes
  int* end;                        // [B,Tb] bucket starts after the scan, bucket ends after the scatter
  T* xs;                           // [C][B*N] coordinates in cell order (graph b at b*N)
  int* idx;                        // [B*N]    node index in cell order
  int32_t* out_idx;                // [B,N,k]
  uint8_t* out_ok;                 // [B,N,k] or null (then empty slots hold -1)
  int32_t* out_count;              // [B,N] in-radius nodes per row, or null
};

// Axis c of graph b's grid: n[c] > 0 cells of width w[c] on a periodic axis of length L[c]; n[c] = 0 on an aperiodic one.
template <typename T, int CD, int PBC>
__device__ __forceinline__ void axis_grids(const RadArgs<T>& a, int b, double (&L)[CD], double (&w)[CD], int (&n)[CD]) {
#pragma unroll
  for (int c = 0; c < CD; ++c) {
    L[c] = 0.0; w[c] = a.cs; n[c] = 0;
    if constexpr (PBC) {
      const T l = a.box[(size_t)b * CD + c];
      if (l > T(0) && l < T(INFINITY)) {
        const double ld = (double)l;
        const double q = fmin(fmax(floor(ld / a.cs), 1.0), RS_CLAMP);
        L[c] = ld; n[c] = (int)q; w[c] = ld / q;
      }
    }
  }
}

__device__ __forceinline__ int cell_coord(double x, double cs, double L, double w, int n) {
  if (n == 0) return (int)fmin(fmax(floor(x / cs), -RS_CLAMP), RS_CLAMP);
  const double p = x - L * floor(x / L);               // wrapped into [0, L] (L itself by rounding: clamped below)
  const int q = (int)floor(p / w);
  return q < 0 ? 0 : (q >= n ? n - 1 : q);
}

template <int CD>
__device__ __forceinline__ int cell_bucket(const int (&cc)[CD], int Tb) {
  unsigned h = (unsigned)cc[0] * 0x8da6b343u;
  if (CD > 1) h ^= (unsigned)cc[CD > 1 ? 1 : 0] * 0xd8163841u;
  if (CD > 2) h ^= (unsigned)cc[CD > 2 ? 2 : 0] * 0xcb1ab31fu;
  h ^= h >> 16; h *= 0x7feb352du;
  h ^= h >> 15; h *= 0x846ca68bu;
  h ^= h >> 16;
  return (int)(h & (unsigned)(Tb - 1));
}

// Node t = b*N + i: its coordinates and whether it goes into the grid (mask set, every coordinate finite).
template <typename T, int CD>
__device__ __forceinline__ bool load_node(const RadArgs<T>& a, size_t t, T (&x)[CD]) {
  bool ok = a.mask ? a.mask[t] != 0 : true;
#pragma unroll
  for (int c = 0; c < CD; ++c) {
    x[c] = a.coors[t * CD + c];
    ok = ok && isfinite(x[c]);
  }
  return ok;
}

// PBC_CELL: the cell coordinates cc of x in graph b's grid, and the cell count n of every axis (0: aperiodic).  A
// periodic axis k is binned in the fractional coordinate s_k = sum_d x_d G[d][k], G = A^-1 of the lower-triangular cell
// A with 1 in place of every aperiodic diagonal, wrapped into [0, 1) and cut into n_k = max(1, floor(w_k / cs)) cells,
// w_k = 1 / |column k of G| being the cell's perpendicular width along a_k.  An aperiodic axis (its row and column of
// A are zero but for the diagonal, so s_k = x_k) is binned as without a cell.  Double precision throughout.
template <typename T, int CD>
__device__ __forceinline__ void frac_cells(const RadArgs<T>& a, int b, const T (&x)[CD], int (&cc)[CD], int (&n)[CD]) {
  const T* m = a.box + (size_t)b * CD * CD;
  double A[CD][CD], G[CD][CD];
  bool per[CD];
#pragma unroll
  for (int r = 0; r < CD; ++r) {
#pragma unroll
    for (int c = 0; c < CD; ++c) { A[r][c] = c <= r ? (double)m[r * CD + c] : 0.0; G[r][c] = 0.0; }
    per[r] = A[r][r] > 0.0 && A[r][r] < INFINITY;
    if (!per[r]) A[r][r] = 1.0;
  }
#pragma unroll
  for (int k = 0; k < CD; ++k) {                       // column k of G: forward substitution down the rows
    G[k][k] = 1.0 / A[k][k];
#pragma unroll
    for (int r = k + 1; r < CD; ++r) {
      double acc = 0.0;
#pragma unroll
      for (int q = k; q < r; ++q) acc = fma(A[r][q], G[q][k], acc);
      G[r][k] = -acc / A[r][r];
    }
  }
#pragma unroll
  for (int k = 0; k < CD; ++k) {
    double s = 0.0, g2 = 0.0;
#pragma unroll
    for (int d = k; d < CD; ++d) { s = fma((double)x[d], G[d][k], s); g2 = fma(G[d][k], G[d][k], g2); }
    n[k] = per[k] ? (int)fmin(fmax(floor(1.0 / (sqrt(g2) * a.cs)), 1.0), RS_CLAMP) : 0;
    cc[k] = n[k] > 0 ? cell_coord(s, a.cs, 1.0, 1.0 / n[k], n[k]) : cell_coord(s, a.cs, 0.0, a.cs, 0);
  }
}

template <typename T, int CD, int PBC>
__device__ __forceinline__ int node_bucket(const RadArgs<T>& a, int b, const T (&x)[CD]) {
  double L[CD], w[CD];
  int n[CD], cc[CD];
  if constexpr (PBC == PBC_CELL) {
    frac_cells<T, CD>(a, b, x, cc, n);
    return cell_bucket<CD>(cc, a.Tb);
  }
  axis_grids<T, CD, PBC>(a, b, L, w, n);
#pragma unroll
  for (int c = 0; c < CD; ++c) cc[c] = cell_coord((double)x[c], a.cs, L[c], w[c], n[c]);
  return cell_bucket<CD>(cc, a.Tb);
}

template <typename T, int CD, int PBC>
__global__ void __launch_bounds__(RS_THREADS) radius_count_kernel(const RadArgs<T> a) {
  const size_t t = (size_t)blockIdx.x * RS_THREADS + threadIdx.x;
  if (t >= (size_t)a.B * a.N) return;
  const int b = (int)(t / a.N), i = (int)(t % a.N);
  T x[CD];
  if (!load_node<T, CD>(a, t, x)) {                   // not in the grid: its row is empty
    for (int s = 0; s < a.k; ++s) {
      a.out_idx[t * a.k + s] = a.out_ok ? i : -1;
      if (a.out_ok) a.out_ok[t * a.k + s] = 0;
    }
    if (a.out_count) a.out_count[t] = 0;
    return;
  }
  atomicAdd(a.cnt + (size_t)b * a.Tb + node_bucket<T, CD, PBC>(a, b, x), 1);
}

__global__ void __launch_bounds__(RS_SCAN_THREADS) radius_scan_kernel(const int* __restrict__ cnt, int* __restrict__ start, int Tb) {
  using Scan = cub::BlockScan<int, RS_SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const size_t g = (size_t)blockIdx.x * Tb;
  int carry = 0;
  for (int base = 0; base < Tb; base += 4 * RS_SCAN_THREADS) {
    int v[4], s = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int t = base + 4 * threadIdx.x + q;
      v[q] = t < Tb ? cnt[g + t] : 0;
      s += v[q];
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(s, excl, total);
    int run = carry + excl;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int t = base + 4 * threadIdx.x + q;
      if (t < Tb) start[g + t] = run;
      run += v[q];
    }
    carry += total;
    __syncthreads();                                   // tmp is reused by the next tile
  }
}

template <typename T, int CD, int PBC>
__global__ void __launch_bounds__(RS_THREADS) radius_scatter_kernel(const RadArgs<T> a) {
  const size_t t = (size_t)blockIdx.x * RS_THREADS + threadIdx.x;
  if (t >= (size_t)a.B * a.N) return;
  const int b = (int)(t / a.N), i = (int)(t % a.N);
  T x[CD];
  if (!load_node<T, CD>(a, t, x)) return;
  const size_t g0 = (size_t)b * a.N, BN = (size_t)a.B * a.N;
  const int pos = atomicAdd(a.end + (size_t)b * a.Tb + node_bucket<T, CD, PBC>(a, b, x), 1);
#pragma unroll
  for (int c = 0; c < CD; ++c) a.xs[c * BN + g0 + pos] = x[c];
  a.idx[g0 + pos] = i;
}

// The candidate stream of node i of graph b, which its warp reads t = lane, lane + 32, ...: the deduplicated buckets of
// the 3^C cells around xi, flattened.  Returns its length; wexcl / wdelta (the warp's 32 ints each) receive per kept
// bucket its first stream position and its cell-order position minus that.
template <typename T, int CD, int PBC>
__device__ __forceinline__ int row_stream(const RadArgs<T>& a, int b, int lane, const T (&xi)[CD], const int* cnt,
                                          const int* end, int* wexcl, int* wdelta) {
  constexpr int NB = CD == 1 ? 3 : (CD == 2 ? 9 : 27);           // neighbouring cells
  // lane l < NB: the bucket of neighbouring cell l; a bucket reached twice (a periodic axis of 1 or 2 cells, or two cells
  // hashing alike) is kept by its lowest lane only, so that no node enters the stream twice
  int bkt = -1 - lane;
  if (lane < NB) {
    double L[CD], w[CD];
    int n[CD], cc[CD];
    int r = lane;
    if constexpr (PBC == PBC_CELL) {
      frac_cells<T, CD>(a, b, xi, cc, n);
#pragma unroll
      for (int c = 0; c < CD; ++c) {
        int v = cc[c] + r % 3 - 1;
        r /= 3;
        if (n[c] > 0) v = v < 0 ? v + n[c] : (v >= n[c] ? v - n[c] : v);
        cc[c] = v;
      }
    } else {
      axis_grids<T, CD, PBC>(a, b, L, w, n);
#pragma unroll
      for (int c = 0; c < CD; ++c) {
        int v = cell_coord((double)xi[c], a.cs, L[c], w[c], n[c]) + r % 3 - 1;
        r /= 3;
        if (n[c] > 0) v = v < 0 ? v + n[c] : (v >= n[c] ? v - n[c] : v);
        cc[c] = v;
      }
    }
    bkt = cell_bucket<CD>(cc, a.Tb);
  }
  const unsigned same = __match_any_sync(0xffffffffu, bkt);
  const bool keep = lane < NB && __ffs(same) - 1 == lane;
  int len = 0, beg = 0;
  if (keep) { len = cnt[bkt]; beg = end[bkt] - len; }
  int incl = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  wexcl[lane] = incl - len;
  wdelta[lane] = beg - (incl - len);
  __syncwarp();
  return total;
}

// Candidate t of the stream: its node index j and its rank, as the all-pairs select computes it (bl / binv: the box of
// graph b under PBC_BOX, pc: its staged cell under PBC_CELL).
template <typename T, int CD, int PBC>
__device__ __forceinline__ T stream_rank(const RadArgs<T>& a, size_t g0, size_t BN, int t, const int* wexcl,
                                         const int* wdelta, const T (&xi)[CD], const T (&bl)[CD], const T (&binv)[CD],
                                         const T* pc, int& j) {
  int s = 0;                                                     // the last kept bucket that starts at or before t
#pragma unroll
  for (int step = 16; step > 0; step >>= 1)
    if (wexcl[s + step] <= t) s += step;
  const size_t pos = g0 + wdelta[s] + t;
  j = a.idx[pos];
  T d = T(0);
  if constexpr (PBC == PBC_CELL) {
    T r[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = c < CD ? xi[c < CD ? c : 0] - a.xs[(c < CD ? c : 0) * BN + pos] : T(0);
    cell_wrap<T>(r[0], r[1], r[2], pc);
#pragma unroll
    for (int c = 0; c < CD; ++c) d = sq_acc<T>(r[c], d);
  } else {
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      T r = xi[c] - a.xs[c * BN + pos];
      if constexpr (PBC) r = min_image<T>(r, bl[c], binv[c]);
      d = sq_acc<T>(r, d);
    }
  }
  return d;
}

// The prologue of both query kernels: the node at cell-order position p of graph b (false: beyond the nodes the graph
// put into its grid), its coordinates xi and its graph's box (bl, binv) or cell (pc).
#define RS_QUERY_ROW()                                                                                                  \
  const int* cnt = a.cnt + (size_t)b * a.Tb;                                                                            \
  const int* end = a.end + (size_t)b * a.Tb;                                                                            \
  if (p >= end[a.Tb - 1]) return;                                                                                       \
  const size_t g0 = (size_t)b * a.N, BN = (size_t)a.B * a.N;                                                            \
  const int i = a.idx[g0 + p];                                                                                          \
  T xi[CD];                                                                                                             \
  _Pragma("unroll") for (int c = 0; c < CD; ++c) xi[c] = a.xs[c * BN + g0 + p];                                         \
  T bl[CD], binv[CD], pc[PBC == PBC_CELL ? CELL_STAGED : 1];                                                            \
  if constexpr (PBC == PBC_CELL) {                                                                                      \
    _Pragma("unroll") for (int t = 0; t < CELL_STAGED; ++t) pc[t] = cell_staged<T>(a.box, b, CD, t);                    \
  } else if constexpr (PBC) {                                                                                           \
    _Pragma("unroll") for (int c = 0; c < CD; ++c) box_axis<T>(a.box, b, CD, c, bl[c], binv[c]);                        \
  }

// k <= 32: lane l keeps the l-th smallest (rank, j) so far; candidates in radius that beat the k-th are queued and merged
// 32 at a time (warp_merge).
template <typename T, int CD, int PBC>
__global__ void __launch_bounds__(RS_WARPS * 32) radius_query_kernel(const RadArgs<T> a) {
  __shared__ T qkey[RS_WARPS][64];
  __shared__ int qidx[RS_WARPS][64];
  __shared__ int sexcl[RS_WARPS][32];
  __shared__ int sdelta[RS_WARPS][32];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const size_t gw = (size_t)blockIdx.x * RS_WARPS + warp;
  if (gw >= (size_t)a.B * a.N) return;
  const int b = (int)(gw / a.N), p = (int)(gw % a.N);
  RS_QUERY_ROW()
  const int total = row_stream<T, CD, PBC>(a, b, lane, xi, cnt, end, sexcl[warp], sdelta[warp]);

  const T INF = T(INFINITY);
  const int IMAX = 0x7fffffff;
  T* myqk = qkey[warp];
  int* myqi = qidx[warp];
  T bkey = INF; int bidx = IMAX;       // lane l: l-th smallest so far
  T thr_key = INF; int thr_idx = IMAX; // the k-th smallest so far
  int count = 0;                       // queued candidates (warp-uniform)
  int nin = 0;                         // this lane's in-radius candidates
  for (int t0 = 0; t0 < total; t0 += 32) {
    const int t = t0 + lane;
    T key = INF;
    int j = IMAX;
    bool pass = false;
    if (t < total) {
      const T d = stream_rank<T, CD, PBC>(a, g0, BN, t, sexcl[warp], sdelta[warp], xi, bl, binv, pc, j);
      const bool in = d <= a.r2;
      nin += in ? 1 : 0;
      key = d;
      pass = in && lex_less<T>(d, j, thr_key, thr_idx);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, pass);
    if (bal == 0) continue;
    if (pass) {
      const int q = count + __popc(bal & ((1u << lane) - 1));
      myqk[q] = key;
      myqi[q] = j;
    }
    count += __popc(bal);
    __syncwarp();
    if (count >= 32) {
      T ckey = myqk[lane];
      int cidx = myqi[lane];
      __syncwarp();
      if (lane + 32 < count) {         // shift the tail of the queue down
        T tk = myqk[lane + 32]; int ti = myqi[lane + 32];
        myqk[lane] = tk; myqi[lane] = ti;
      }
      count -= 32;
      __syncwarp();
      warp_merge<T>(bkey, bidx, ckey, cidx, lane);
      thr_key = shfl_idx_t<T>(bkey, a.k - 1);
      thr_idx = __shfl_sync(0xffffffffu, bidx, a.k - 1);
    }
  }
  if (count > 0) {
    T ckey = lane < count ? myqk[lane] : INF;
    int cidx = lane < count ? myqi[lane] : IMAX;
    warp_merge<T>(bkey, bidx, ckey, cidx, lane);
  }
  const size_t row = g0 + i;
  if (lane < a.k) {
    const size_t o = row * a.k + lane;
    const bool kept = bidx != IMAX;
    a.out_idx[o] = kept ? bidx : (a.out_ok ? i : -1);
    if (a.out_ok) a.out_ok[o] = kept ? 1 : 0;
  }
  if (a.out_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nin += __shfl_xor_sync(0xffffffffu, nin, o);
    if (lane == 0) a.out_count[row] = nin;
  }
}

// Sorts n = 2^m (rank, j) pairs in shared memory ascending (lexicographic), one warp: the bitonic network of
// knn_block_sort_kernel.
template <typename T>
__device__ __forceinline__ void warp_smem_sort(T* key, int* idx, int n, int lane) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = lane; t < n / 2; t += 32) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const bool asc = (lo & size) == 0;
        if (lex_less<T>(key[hi], idx[hi], key[lo], idx[lo]) == asc) {
          const T tk = key[lo]; key[lo] = key[hi]; key[hi] = tk;
          const int ti = idx[lo]; idx[lo] = idx[hi]; idx[hi] = ti;
        }
      }
      __syncwarp();
    }
  }
}

// 32 < k <= RS_WIDE_MAX_K: the candidate stream of radius_query_kernel, with the top k kept in shared memory instead of
// lanes.  Per warp, KP = next_pow2(k) (>= 64) pairs `list`, sorted ascending (the KP smallest (rank, j) so far, padded
// with (inf, IMAX)), and KP more `queue`.  A candidate in radius that beats the current k-th list entry is queued.  Once
// the queue could not take another 32, it is padded, sorted and merged into the list: list[s] = min(list[s],
// queue[KP-1-s]) leaves the KP smallest of both as a bitonic sequence, which log2(KP) merge steps sort.  The list is a
// function of the set of pairs queued, and every pair the filter drops is beaten by k listed ones, so the k kept pairs
// are the k smallest of the stream whatever order the scatter put the candidates in.
template <typename T, int CD, int PBC>
__global__ void __launch_bounds__(RS_WARPS * 32) radius_query_wide_kernel(const RadArgs<T> a, int KP) {
  extern __shared__ __align__(16) unsigned char rsw_sm[];         // [warps][2 KP] ranks, then [warps][2 KP] indices
  __shared__ int sexcl[RS_WARPS][32];
  __shared__ int sdelta[RS_WARPS][32];
  const int warps = blockDim.x / 32, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const size_t gw = (size_t)blockIdx.x * warps + warp;
  if (gw >= (size_t)a.B * a.N) return;
  const int b = (int)(gw / a.N), p = (int)(gw % a.N);
  RS_QUERY_ROW()
  const int total = row_stream<T, CD, PBC>(a, b, lane, xi, cnt, end, sexcl[warp], sdelta[warp]);

  const T INF = T(INFINITY);
  const int IMAX = 0x7fffffff;
  T* lk = reinterpret_cast<T*>(rsw_sm) + (size_t)warp * 2 * KP;
  int* li = reinterpret_cast<int*>(reinterpret_cast<T*>(rsw_sm) + (size_t)warps * 2 * KP) + (size_t)warp * 2 * KP;
  T* qk = lk + KP;
  int* qi = li + KP;
  for (int s = lane; s < KP; s += 32) { lk[s] = INF; li[s] = IMAX; }
  T thr_key = INF; int thr_idx = IMAX; // the k-th smallest so far
  int count = 0;                       // queued candidates (warp-uniform)
  int nin = 0;                         // this lane's in-radius candidates
  auto flush = [&]() {
    for (int s = count + lane; s < KP; s += 32) { qk[s] = INF; qi[s] = IMAX; }
    __syncwarp();
    warp_smem_sort<T>(qk, qi, KP, lane);
    for (int s = lane; s < KP; s += 32) {
      const T ck = qk[KP - 1 - s];
      const int ci = qi[KP - 1 - s];
      if (lex_less<T>(ck, ci, lk[s], li[s])) { lk[s] = ck; li[s] = ci; }
    }
    __syncwarp();
    for (int stride = KP >> 1; stride > 0; stride >>= 1) {
      for (int t = lane; t < KP / 2; t += 32) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        if (lex_less<T>(lk[hi], li[hi], lk[lo], li[lo])) {
          const T tk = lk[lo]; lk[lo] = lk[hi]; lk[hi] = tk;
          const int ti = li[lo]; li[lo] = li[hi]; li[hi] = ti;
        }
      }
      __syncwarp();
    }
    count = 0;
    thr_key = lk[a.k - 1];
    thr_idx = li[a.k - 1];
  };
  for (int t0 = 0; t0 < total; t0 += 32) {
    const int t = t0 + lane;
    T key = INF;
    int j = IMAX;
    bool pass = false;
    if (t < total) {
      key = stream_rank<T, CD, PBC>(a, g0, BN, t, sexcl[warp], sdelta[warp], xi, bl, binv, pc, j);
      const bool in = key <= a.r2;
      nin += in ? 1 : 0;
      pass = in && lex_less<T>(key, j, thr_key, thr_idx);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, pass);
    if (bal == 0) continue;
    if (pass) {
      const int q = count + __popc(bal & ((1u << lane) - 1));
      qk[q] = key;
      qi[q] = j;
    }
    count += __popc(bal);
    if (count > KP - 32) flush();
  }
  if (count > 0) flush();
  const size_t row = g0 + i;
  for (int s = lane; s < a.k; s += 32) {
    const size_t o = row * a.k + s;
    const bool kept = li[s] != IMAX;
    a.out_idx[o] = kept ? li[s] : (a.out_ok ? i : -1);
    if (a.out_ok) a.out_ok[o] = kept ? 1 : 0;
  }
  if (a.out_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nin += __shfl_xor_sync(0xffffffffu, nin, o);
    if (lane == 0) a.out_count[row] = nin;
  }
}

template <typename T, int CD, int PBC>
static int launch_cell(const RadArgs<T>& a, cudaStream_t st) {
  const size_t nodes = (size_t)a.B * a.N;
  const unsigned gn = (unsigned)((nodes + RS_THREADS - 1) / RS_THREADS);
  EGNN_CUDA_TRY(cudaMemsetAsync(a.cnt, 0, (size_t)a.B * a.Tb * sizeof(int), st));
  radius_count_kernel<T, CD, PBC><<<gn, RS_THREADS, 0, st>>>(a);
  EGNN_LAUNCH_CHECK();
  radius_scan_kernel<<<a.B, RS_SCAN_THREADS, 0, st>>>(a.cnt, a.end, a.Tb);
  EGNN_LAUNCH_CHECK();
  radius_scatter_kernel<T, CD, PBC><<<gn, RS_THREADS, 0, st>>>(a);
  EGNN_LAUNCH_CHECK();
  if (a.k <= 32) {
    radius_query_kernel<T, CD, PBC><<<(unsigned)((nodes + RS_WARPS - 1) / RS_WARPS), RS_WARPS * 32, 0, st>>>(a);
  } else {
    int KP = 64;
    while (KP < a.k) KP <<= 1;
    const size_t per_warp = (size_t)2 * KP * (sizeof(T) + sizeof(int));
    const int warps = per_warp * RS_WARPS <= RS_WIDE_SMEM ? RS_WARPS : RS_WARPS / 2;      // fp64 at k > 128: 4 warps
    radius_query_wide_kernel<T, CD, PBC><<<(unsigned)((nodes + warps - 1) / warps), warps * 32, warps * per_warp, st>>>(
        a, KP);
  }
  EGNN_LAUNCH_CHECK();
  count_launch(4);
  return EGNN_OK;
}

template <typename T>
static int cell_select(int B, int N, int C, int k, const void* coors, const uint8_t* mask, const void* box, double r2,
                       int32_t* out_idx, uint8_t* out_ok, int32_t* out_count, void* ws, cudaStream_t st, int pbc) {
  const CellWs L = cell_ws_layout(B, N, C, sizeof(T));
  char* base = static_cast<char*>(ws);
  RadArgs<T> a;
  a.B = B; a.N = N; a.k = k; a.Tb = rs_buckets(N);
  a.r2 = (T)r2;
  a.cs = sqrt((double)a.r2) * (1.0 + 0x1p-10);
  a.coors = static_cast<const T*>(coors); a.mask = mask; a.box = static_cast<const T*>(box);
  a.cnt = reinterpret_cast<int*>(base + L.cnt);
  a.end = reinterpret_cast<int*>(base + L.end);
  a.xs = reinterpret_cast<T*>(base + L.xs);
  a.idx = reinterpret_cast<int*>(base + L.idx);
  a.out_idx = out_idx; a.out_ok = out_ok; a.out_count = out_count;
  if (box && pbc == PBC_CELL) {
    if (C == 2) return launch_cell<T, 2, PBC_CELL>(a, st);
    if (C == 3) return launch_cell<T, 3, PBC_CELL>(a, st);
    return EGNN_ERR_SHAPE;
  }
  switch (C * 2 + (box ? 1 : 0)) {
    case 2: return launch_cell<T, 1, PBC_NONE>(a, st);
    case 3: return launch_cell<T, 1, PBC_BOX>(a, st);
    case 4: return launch_cell<T, 2, PBC_NONE>(a, st);
    case 5: return launch_cell<T, 2, PBC_BOX>(a, st);
    case 6: return launch_cell<T, 3, PBC_NONE>(a, st);
    case 7: return launch_cell<T, 3, PBC_BOX>(a, st);
    default: return EGNN_ERR_UNSUPPORTED;
  }
}

static int radius_check(int B, int N, int C, int k, int max_k) {
  if (B <= 0 || N <= 0 || C <= 0 || k <= 0 || k > N) return EGNN_ERR_SHAPE;
  if (k > max_k || C > 3) return EGNN_ERR_UNSUPPORTED;
  if ((long long)B * rs_buckets(N) > 0x7fffffffLL) return EGNN_ERR_SHAPE;    // int bucket and node offsets
  return EGNN_OK;
}

// r2 is the radius as the caller passes it; the kernels compare against (T)r2.  k up to RS_WIDE_MAX_K: the callers bound
// it (egnn_radius_select at 32, cell_select_eligible by the descriptor's flags).
int cell_select_dispatch(int32_t dtype, int B, int N, int C, int k, const void* coors, const uint8_t* mask,
                         const void* box, double r2, int32_t* out_idx, uint8_t* out_ok, int32_t* out_count, void* ws,
                         cudaStream_t st, int pbc) {
  if (!coors || !out_idx || !ws) return EGNN_ERR_NULL;
  EGNN_TRY(radius_check(B, N, C, k, RS_WIDE_MAX_K));
  if (dtype == EGNN_DTYPE_F64) {
    if (!(r2 > 0.0)) return EGNN_ERR_SHAPE;
    return cell_select<double>(B, N, C, k, coors, mask, box, r2, out_idx, out_ok, out_count, ws, st, pbc);
  }
  if (dtype != EGNN_DTYPE_F32) return EGNN_ERR_UNSUPPORTED;
  if (!((float)r2 > 0.f)) return EGNN_ERR_SHAPE;
  return cell_select<float>(B, N, C, k, coors, mask, box, r2, out_idx, out_ok, out_count, ws, st, pbc);
}

// The public entries: egnn_radius_select* with k <= 32, egnn_radius_select_wide* with k <= RS_WIDE_MAX_K.
static int radius_ws_entry(int max_k, int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes) {
  if (!out_bytes) return EGNN_ERR_NULL;
  EGNN_TRY(radius_check(B, N, C, k, max_k));
  *out_bytes = cell_select_ws_bytes(B, N, C, 8);               // sized for float64 coordinates: covers both types
  return EGNN_OK;
}

// lattice: a [B,C] box (pbc = PBC_BOX, may be null) or a [B,C,C] cell (PBC_CELL)
static int radius_entry(int max_k, int pbc, int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                        const uint8_t* mask, const void* lattice, double r2, int32_t* out_idx, int32_t* out_count,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (!workspace || (pbc == PBC_CELL && !lattice)) return EGNN_ERR_NULL;
  if (pbc == PBC_CELL && (C < 2 || C > 3)) return EGNN_ERR_SHAPE;    // a cell is 2-D or 3-D (before radius_check's C > 3)
  EGNN_TRY(radius_check(B, N, C, k, max_k));
  if ((uintptr_t)workspace & 0xFF) return EGNN_ERR_ALIGN;
  if (workspace_bytes < cell_select_ws_bytes(B, N, C, dtype == EGNN_DTYPE_F64 ? 8 : 4)) return EGNN_ERR_WORKSPACE;
  return cell_select_dispatch(dtype, B, N, C, k, coors, mask, lattice, r2, out_idx, nullptr, out_count, workspace,
                              static_cast<cudaStream_t>(stream), pbc);
}

}  // namespace egnn

extern "C" int egnn_radius_select_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes) {
  return egnn::radius_ws_entry(32, B, N, C, k, out_bytes);
}

extern "C" int egnn_radius_select(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                  const uint8_t* mask, const void* box, double r2, int32_t* out_idx, int32_t* out_count,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  return egnn::radius_entry(32, egnn::PBC_BOX, dtype, B, N, C, k, coors, mask, box, r2, out_idx, out_count, workspace,
                            workspace_bytes, stream);
}

extern "C" int egnn_radius_select_triclinic(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                            const uint8_t* mask, const void* cell, double r2, int32_t* out_idx,
                                            int32_t* out_count, void* workspace, size_t workspace_bytes, void* stream) {
  return egnn::radius_entry(32, egnn::PBC_CELL, dtype, B, N, C, k, coors, mask, cell, r2, out_idx, out_count, workspace,
                            workspace_bytes, stream);
}

extern "C" int egnn_radius_select_wide_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes) {
  return egnn::radius_ws_entry(egnn::RS_WIDE_MAX_K, B, N, C, k, out_bytes);
}

extern "C" int egnn_radius_select_wide(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                       const uint8_t* mask, const void* box, double r2, int32_t* out_idx,
                                       int32_t* out_count, void* workspace, size_t workspace_bytes, void* stream) {
  return egnn::radius_entry(egnn::RS_WIDE_MAX_K, egnn::PBC_BOX, dtype, B, N, C, k, coors, mask, box, r2, out_idx,
                            out_count, workspace, workspace_bytes, stream);
}

extern "C" int egnn_radius_select_wide_triclinic(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k,
                                                 const void* coors, const uint8_t* mask, const void* cell, double r2,
                                                 int32_t* out_idx, int32_t* out_count, void* workspace,
                                                 size_t workspace_bytes, void* stream) {
  return egnn::radius_entry(egnn::RS_WIDE_MAX_K, egnn::PBC_CELL, dtype, B, N, C, k, coors, mask, cell, r2, out_idx,
                            out_count, workspace, workspace_bytes, stream);
}

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
// A triclinic cell bins its periodic axes in fractional coordinates instead (radius_cells).
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
//
// The kNN grid (egnn_knn_grid_select, the second half of this file) answers the plain k-nearest query with no cutoff on
// the same count / scan / scatter, with a dense grid whose cell edge each graph sizes on the device from its extent
// (knn_grid_setup_kernel), and a query that visits Chebyshev rings of cells until no unvisited node can rank before
// the k-th (knn_ring_kernel).  Rows the grid cannot decide are ranked against every node of their graph
// (knn_scan_kernel); padded rows are written directly.  Its lists equal egnn_knn_select's bit for bit (DESIGN.md
// section 5).
#include "common.cuh"
#include "profile.h"
#include "warp_select.cuh"
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

namespace egnn {

constexpr int RS_THREADS = 256;          // count / scatter
constexpr int RS_SCAN_THREADS = 1024;    // scan: one CTA per graph, 4 buckets per thread per tile
constexpr int RS_WARPS = 8;              // query rows per CTA
constexpr int RS_WIDE_MAX_K = 256;       // the longest list the query keeps (radius_query_wide_kernel above 32)
constexpr size_t RS_WIDE_SMEM = 32768;   // wide query: dynamic shared memory per CTA, within the 48 KiB default
constexpr double RS_CLAMP = 1073741824.0;     // 2^30: aperiodic cell coordinates and periodic cell counts
constexpr int GRID_RADIUS = 0, GRID_KNN = 1;  // which grid the count / scatter kernels bin into

// Buckets per graph: next_pow2(2N).
__host__ __device__ inline int rs_buckets(int N) {
  int t = 2;
  while (t < 2 * N) t <<= 1;
  return t;
}

// The grid's scratch from byte `o` on, for `nodes` nodes in `nb` buckets: B N nodes in B next_pow2(2N) buckets, or
// the T nodes of a packed batch in 4 T buckets (graph g's from 4 ptr[g] on, next_pow2(2 n_g) <= 4 n_g of them).
struct CellWs { size_t cnt, end, xs, idx, total; };
static CellWs cell_ws_layout(size_t nodes, size_t nb, int C, size_t coord_bytes, size_t o = 0) {
  CellWs w;
  auto take = [&](size_t bytes) { size_t r = o; o += round_up(bytes, 256); return r; };
  w.cnt = take(nb * sizeof(int));
  w.end = take(nb * sizeof(int));
  w.xs = take((size_t)C * nodes * coord_bytes);
  w.idx = take(nodes * sizeof(int));
  w.total = o;
  return w;
}

// The kNN grid of one graph, set by knn_grid_setup_kernel and read by every later launch (no host round trip).
// Cell coordinate c of a node: on an aperiodic axis floor((x_c - lo[c]) / cs), in [0, n[c]); on a periodic axis the
// position (x_c, or the fractional coordinate under a cell) wrapped into [0, L[c]) and cut into n[c] cells.
struct KGrid {
  double cs;          // cell edge of the aperiodic axes
  double lo[3];       // aperiodic axis: the smallest coordinate of the graph's insertable nodes
  double L[3];        // periodic axis: the binned period (the box length, or 1 for a fractional coordinate); 0 aperiodic
  double w[3];        // a node one cell further along axis c is at least this much further away (cs, L / n, w_c / n)
  double G[3][3];     // PBC_CELL: the inverse cell (cell_inverse)
  double err;         // absolute rounding allowance of the stopping test
  int n[3];           // cells per axis (1 beyond C); their product is at most Tb
  int ok;             // 0: no usable grid (fewer than k insertable nodes, a non-finite extent): every row is scanned
};
static_assert(sizeof(KGrid) == 176, "KGrid layout");

struct KnnWs { CellWs cell; size_t kg, fb, nfb, total; };
static KnnWs knn_ws_layout(int graphs, size_t nodes, size_t nb, int C, size_t coord_bytes, size_t o = 0) {
  KnnWs w;
  w.cell = cell_ws_layout(nodes, nb, C, coord_bytes, o);
  o = w.cell.total;
  auto take = [&](size_t bytes) { size_t r = o; o += round_up(bytes, 256); return r; };
  w.kg = take((size_t)graphs * sizeof(KGrid));
  w.fb = take(nodes * sizeof(int));
  w.nfb = take(sizeof(int));
  w.total = o;
  return w;
}

// The scratch of the radius grid (GRID_RADIUS) or of the kNN grid (GRID_KNN), which contains the radius grid's.
static size_t grid_ws_bytes(int grid, int B, int N, int C, size_t coord_bytes) {
  const size_t nodes = (size_t)B * N, nb = (size_t)B * rs_buckets(N);
  return grid == GRID_KNN ? knn_ws_layout(B, nodes, nb, C, coord_bytes).total
                          : cell_ws_layout(nodes, nb, C, coord_bytes).total;
}

// The k, C and flags both grids serve: k <= 32, or <= RS_WIDE_MAX_K under EGNN_FLAG_CELL_SELECT_WIDE; C <= 3; no
// only_sparse, batched adjacency or per-slot edges.
static bool grid_eligible(const EgnnLayerDesc& d) {
  const int max_k = (d.flags & EGNN_FLAG_CELL_SELECT_WIDE) ? RS_WIDE_MAX_K : 32;
  if (d.k < 1 || d.k > max_k || d.C < 1 || d.C > 3) return false;
  return !(d.flags & (EGNN_FLAG_ONLY_SPARSE | EGNN_FLAG_ADJ_BATCHED | EGNN_FLAG_EDGES_PER_SLOT));
}

bool cell_select_eligible(const EgnnLayerDesc& d) {
  if (!grid_eligible(d)) return false;
  // the radius in the coordinates' type, as the select compares it; at or above 1e5 padded pairs (rank 1e5) could
  // take slots in the reference
  const double r2 = d.dtype == EGNN_DTYPE_F64 ? d.valid_radius : (double)(float)d.valid_radius;
  return r2 > 0.0 && r2 < 1e5;
}

static bool knn_grid_eligible(const EgnnLayerDesc& d) { return (d.flags & EGNN_FLAG_KNN_GRID) && grid_eligible(d); }

// The radius grid's scratch for a layer it may serve; under EGNN_FLAG_KNN_GRID the kNN grid's, which is larger, for a
// layer the kNN grid may serve (either can run, depending on the call's mask).
size_t cell_select_layer_ws_bytes(const EgnnLayerDesc& d) {
  const size_t cb = d.dtype == EGNN_DTYPE_F64 ? 8 : 4;
  if (knn_grid_eligible(d)) return grid_ws_bytes(GRID_KNN, d.B, d.N, d.C, cb);
  return cell_select_eligible(d) ? grid_ws_bytes(GRID_RADIUS, d.B, d.N, d.C, cb) : 0;
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
  // the kNN grid only
  KGrid* kg;                       // [B]
  int* fb_rows;                    // [B*N] rows (b*N + i) left to knn_scan_kernel
  int* fb_count;                   // their number
  T vr;                            // ok = rank <= vr
  // the segment form (SEG, a packed batch): B = G graphs, N = T nodes; graph b holds nodes [ptr[b], ptr[b+1]) and
  // buckets [4 ptr[b], 4 ptr[b] + next_pow2(2 n_b)), idx holds node-axis indices, and one box or cell serves every graph
  const int32_t* ptr;              // [G+1]
  const int* seg_valid;            // 1: ptr is non-decreasing within [0, T] (seg_grid_tiles_kernel), else no graph is on the grid
  int min_n;                       // graphs of fewer nodes are not on the grid (at least k and 1)
};

// Graph b as the kernels address it: its lattice index lb, bucket count Tb, first node g0 (on the node axis and in
// xs / idx) and first bucket.
struct GraphAt { int b, lb, Tb; size_t g0, bkt; };

template <typename T, bool SEG>
__device__ __forceinline__ GraphAt graph_at(const RadArgs<T>& a, int b) {
  if constexpr (SEG) {
    const int lo = a.ptr[b];
    return {b, 0, rs_buckets(a.ptr[b + 1] - lo), (size_t)lo, 4 * (size_t)lo};
  } else {
    return {b, b, a.Tb, (size_t)b * a.N, (size_t)b * a.Tb};
  }
}

// The fields of g as the unpacked form reads them straight from its arguments (graph b = g.b), so that its kernels
// compile as they did before the segment form.
template <typename T, bool SEG>
__device__ __forceinline__ int tb_of(const RadArgs<T>& a, const GraphAt& g) { return SEG ? g.Tb : a.Tb; }
template <bool SEG>
__device__ __forceinline__ int lb_of(const GraphAt& g) { return SEG ? 0 : g.b; }
template <typename T, bool SEG>
__device__ __forceinline__ size_t bkt_of(const RadArgs<T>& a, const GraphAt& g) {
  return SEG ? g.bkt : (size_t)g.b * a.Tb;
}
template <typename T, bool SEG>
__device__ __forceinline__ size_t g0_of(const RadArgs<T>& a, const GraphAt& g) { return SEG ? g.g0 : (size_t)g.b * a.N; }

// SEG: whether graph b is on the grid (a valid ptr, at least min_n nodes).
template <typename T>
__device__ __forceinline__ bool seg_on_grid(const RadArgs<T>& a, int b) {
  return *a.seg_valid && a.ptr[b + 1] - a.ptr[b] >= a.min_n;
}

// SEG: the graph b holding node t, if it is on the grid (the last b with ptr[b] <= t; ptr is valid).
template <typename T>
__device__ __forceinline__ bool seg_node(const RadArgs<T>& a, int t, int& b) {
  if (!*a.seg_valid) return false;
  int lo = 0, hi = a.B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.ptr[mid] <= t) lo = mid; else hi = mid - 1;
  }
  b = lo;
  return t >= a.ptr[b] && t < a.ptr[b + 1] && a.ptr[b + 1] - a.ptr[b] >= a.min_n;
}

// Nodes on the launch's node axis: B N, or T in the segment form.
template <typename T, bool SEG>
__device__ __forceinline__ size_t grid_nodes(const RadArgs<T>& a) { return SEG ? (size_t)a.N : (size_t)a.B * a.N; }

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

// G = A^-1 of graph b's lower-triangular cell A (m: [CD][CD]) with 1 in place of every aperiodic diagonal (per[r]:
// axis r is periodic); column k of G by forward substitution down the rows, in double.
template <typename T, int CD>
__device__ __forceinline__ void cell_inverse(const T* m, double (&G)[CD][CD], bool (&per)[CD]) {
  double A[CD][CD];
#pragma unroll
  for (int r = 0; r < CD; ++r) {
#pragma unroll
    for (int c = 0; c < CD; ++c) { A[r][c] = c <= r ? (double)m[r * CD + c] : 0.0; G[r][c] = 0.0; }
    per[r] = A[r][r] > 0.0 && A[r][r] < INFINITY;
    if (!per[r]) A[r][r] = 1.0;
  }
#pragma unroll
  for (int k = 0; k < CD; ++k) {
    G[k][k] = 1.0 / A[k][k];
#pragma unroll
    for (int r = k + 1; r < CD; ++r) {
      double acc = 0.0;
#pragma unroll
      for (int q = k; q < r; ++q) acc = fma(A[r][q], G[q][k], acc);
      G[r][k] = -acc / A[r][r];
    }
  }
}

// The cell coordinates cc of x in graph b's radius grid, and the cell count n of every axis (0: aperiodic).  An
// aperiodic axis is cut into cells of edge cs = a.cs.  A periodic box axis of length L has n = max(1, floor(L / cs))
// cells of width L / n >= cs, positions wrapped into [0, L).  Under a cell (PBC_CELL) a periodic axis k is binned in the
// fractional coordinate s_k = sum_d x_d G[d][k] (cell_inverse), wrapped into [0, 1) and cut into
// n_k = max(1, floor(w_k / cs)) cells, w_k = 1 / |column k of G| being the cell's perpendicular width along a_k; an
// aperiodic axis (its row and column of A are zero but for the diagonal, so s_k = x_k) is binned as without a cell.
// Double precision throughout.
template <typename T, int CD, int PBC>
__device__ __forceinline__ void radius_cells(const RadArgs<T>& a, int b, const T (&x)[CD], int (&cc)[CD], int (&n)[CD]) {
  if constexpr (PBC == PBC_CELL) {
    double G[CD][CD];
    bool per[CD];
    cell_inverse<T, CD>(a.box + (size_t)b * CD * CD, G, per);
#pragma unroll
    for (int k = 0; k < CD; ++k) {
      double s = 0.0, g2 = 0.0;
#pragma unroll
      for (int d = k; d < CD; ++d) { s = fma((double)x[d], G[d][k], s); g2 = fma(G[d][k], G[d][k], g2); }
      n[k] = per[k] ? (int)fmin(fmax(floor(1.0 / (sqrt(g2) * a.cs)), 1.0), RS_CLAMP) : 0;
      cc[k] = n[k] > 0 ? cell_coord(s, a.cs, 1.0, 1.0 / n[k], n[k]) : cell_coord(s, a.cs, 0.0, a.cs, 0);
    }
  } else {
    double L[CD], w[CD];
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
#pragma unroll
    for (int c = 0; c < CD; ++c) cc[c] = cell_coord((double)x[c], a.cs, L[c], w[c], n[c]);
  }
}

// Cell coordinates of x in the kNN grid g, each in [0, g.n[c]).
template <typename T, int CD, int PBC>
__device__ __forceinline__ void knn_cell(const KGrid& g, const T (&x)[CD], int (&cc)[CD]) {
#pragma unroll
  for (int c = 0; c < CD; ++c) {
    double s = (double)x[c];
    if constexpr (PBC == PBC_CELL) {
      s = 0.0;
#pragma unroll
      for (int d = c; d < CD; ++d) s = fma((double)x[d], g.G[d][c], s);
    }
    const int n = g.n[c];
    if (g.L[c] > 0.0) cc[c] = cell_coord(s, g.cs, g.L[c], g.L[c] / n, n);
    else cc[c] = (int)fmin(fmax(floor((s - g.lo[c]) / g.cs), 0.0), (double)(n - 1));
  }
}

template <int CD>
__device__ __forceinline__ int knn_index(const KGrid& g, const int (&cc)[CD]) {
  int t = cc[CD - 1];
#pragma unroll
  for (int c = CD - 2; c >= 0; --c) t = t * g.n[c] + cc[c];
  return t;
}

// The bucket node x of graph g goes to, within its region: a hashed radius cell, or a dense kNN cell.
template <typename T, int CD, int PBC, int GRID, bool SEG>
__device__ __forceinline__ int grid_bucket(const RadArgs<T>& a, const GraphAt& g, const T (&x)[CD]) {
  int cc[CD];
  if constexpr (GRID == GRID_KNN) {
    knn_cell<T, CD, PBC>(a.kg[g.b], x, cc);
    return knn_index<CD>(a.kg[g.b], cc);
  } else {
    int n[CD];
    radius_cells<T, CD, PBC>(a, lb_of<SEG>(g), x, cc, n);
    return cell_bucket<CD>(cc, tb_of<T, SEG>(a, g));
  }
}

// Row t = b*N + i of a node the grid does not hold (i = t in the segment form).  The radius grid leaves it empty.  The
// kNN grid writes a padded row (every rank 1e5 in egnn_knn_select: the graph's first k nodes, from node j0, with
// ok = (1e5 <= vr)) and leaves a non-finite node's row to the full scan.
template <typename T, int GRID>
__device__ __forceinline__ void outside_row(const RadArgs<T>& a, size_t t, int i, int j0) {
  if constexpr (GRID == GRID_KNN) {
    if (a.mask && !a.mask[t]) {
      for (int s = 0; s < a.k; ++s) {
        a.out_idx[t * a.k + s] = j0 + s;
        if (a.out_ok) a.out_ok[t * a.k + s] = T(1e5) <= a.vr ? 1 : 0;
      }
    } else {
      a.fb_rows[atomicAdd(a.fb_count, 1)] = (int)t;
    }
  } else {
    for (int s = 0; s < a.k; ++s) {
      a.out_idx[t * a.k + s] = a.out_ok ? i : -1;
      if (a.out_ok) a.out_ok[t * a.k + s] = 0;
    }
    if (a.out_count) a.out_count[t] = 0;
  }
}

// The node (graph b, index i) of thread t: b = t / N, i = t % N; in the segment form (SEG) the graph holding node t,
// i = t, false when that graph is not on the grid.
template <typename T, bool SEG>
__device__ __forceinline__ bool grid_thread_node(const RadArgs<T>& a, size_t t, int& b, int& i) {
  if constexpr (SEG) {
    i = (int)t;
    return seg_node(a, i, b);
  } else {
    b = (int)(t / a.N); i = (int)(t % a.N);
    return true;
  }
}

template <typename T, int CD, int PBC, int GRID = GRID_RADIUS, bool SEG = false>
__global__ void __launch_bounds__(RS_THREADS) radius_count_kernel(const RadArgs<T> a) {
  const size_t t = (size_t)blockIdx.x * RS_THREADS + threadIdx.x;
  if (t >= grid_nodes<T, SEG>(a)) return;
  int b, i;
  if (!grid_thread_node<T, SEG>(a, t, b, i)) return;
  T x[CD];
  if (!load_node<T, CD>(a, t, x)) {                   // not in the grid
    outside_row<T, GRID>(a, t, i, SEG ? a.ptr[b] : 0);
    return;
  }
  const GraphAt g = graph_at<T, SEG>(a, b);
  atomicAdd(a.cnt + bkt_of<T, SEG>(a, g) + grid_bucket<T, CD, PBC, GRID, SEG>(a, g, x), 1);
}

// The exclusive prefix of the Tb bucket sizes cnt[g ..] into start[g ..], by one CTA.
__device__ __forceinline__ void scan_buckets(const int* __restrict__ cnt, int* __restrict__ start, size_t g, int Tb) {
  using Scan = cub::BlockScan<int, RS_SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
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

__global__ void __launch_bounds__(RS_SCAN_THREADS) radius_scan_kernel(const int* __restrict__ cnt, int* __restrict__ start, int Tb) {
  scan_buckets(cnt, start, (size_t)blockIdx.x * Tb, Tb);
}

// The segment form of radius_scan_kernel: graph blockIdx.x's region, if the graph is on the grid.
template <typename T>
__global__ void __launch_bounds__(RS_SCAN_THREADS) radius_scan_seg_kernel(const RadArgs<T> a) {
  if (!seg_on_grid(a, blockIdx.x)) return;
  const GraphAt g = graph_at<T, true>(a, blockIdx.x);
  scan_buckets(a.cnt, a.end, g.bkt, g.Tb);
}

template <typename T, int CD, int PBC, int GRID = GRID_RADIUS, bool SEG = false>
__global__ void __launch_bounds__(RS_THREADS) radius_scatter_kernel(const RadArgs<T> a) {
  const size_t t = (size_t)blockIdx.x * RS_THREADS + threadIdx.x;
  if (t >= grid_nodes<T, SEG>(a)) return;
  int b, i;
  if (!grid_thread_node<T, SEG>(a, t, b, i)) return;
  T x[CD];
  if (!load_node<T, CD>(a, t, x)) return;
  const GraphAt g = graph_at<T, SEG>(a, b);
  const size_t g0 = g0_of<T, SEG>(a, g), BN = grid_nodes<T, SEG>(a);
  const int pos = atomicAdd(a.end + bkt_of<T, SEG>(a, g) + grid_bucket<T, CD, PBC, GRID, SEG>(a, g, x), 1);
#pragma unroll
  for (int c = 0; c < CD; ++c) a.xs[c * BN + g0 + pos] = x[c];
  a.idx[g0 + pos] = i;
}

// The stream of the buckets the warp's lanes hold (bkt, where keep is set), flattened in lane order: returns its
// length; wexcl / wdelta receive per lane its bucket's first stream position and its cell-order position minus that.
__device__ __forceinline__ int bucket_stream(int lane, bool keep, int bkt, const int* cnt, const int* end, int* wexcl,
                                             int* wdelta) {
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

// The candidate stream of node i of graph b, which its warp reads t = lane, lane + 32, ...: the deduplicated buckets of
// the 3^C cells around xi, flattened.  Returns its length; wexcl / wdelta (the warp's 32 ints each) receive per kept
// bucket its first stream position and its cell-order position minus that.
template <typename T, int CD, int PBC, bool SEG>
__device__ __forceinline__ int row_stream(const RadArgs<T>& a, const GraphAt& g, int lane, const T (&xi)[CD],
                                          const int* cnt, const int* end, int* wexcl, int* wdelta) {
  constexpr int NB = CD == 1 ? 3 : (CD == 2 ? 9 : 27);           // neighbouring cells
  // lane l < NB: the bucket of neighbouring cell l; a bucket reached twice (a periodic axis of 1 or 2 cells, or two cells
  // hashing alike) is kept by its lowest lane only, so that no node enters the stream twice
  int bkt = -1 - lane;
  if (lane < NB) {
    int n[CD], cc[CD];
    radius_cells<T, CD, PBC>(a, lb_of<SEG>(g), xi, cc, n);
    int r = lane;
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      int v = cc[c] + r % 3 - 1;
      r /= 3;
      if (n[c] > 0) v = v < 0 ? v + n[c] : (v >= n[c] ? v - n[c] : v);
      cc[c] = v;
    }
    bkt = cell_bucket<CD>(cc, tb_of<T, SEG>(a, g));
  }
  const unsigned same = __match_any_sync(0xffffffffu, bkt);
  return bucket_stream(lane, lane < NB && __ffs(same) - 1 == lane, bkt, cnt, end, wexcl, wdelta);
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
  return pair_rank<T, CD, PBC>(xi, [&](int c) { return a.xs[c * BN + pos]; }, CD, bl, binv, pc);
}

// The graph and cell-order position of the query warp gw: graph gw / N, position gw % N; in the segment form (SEG)
// the graph holding node gw (its region of xs / idx is its node range), false when that graph is not on the grid.
template <typename T, bool SEG>
__device__ __forceinline__ bool grid_query_row(const RadArgs<T>& a, size_t gw, GraphAt& g, int& p) {
  int b;
  if constexpr (SEG) {
    if (!seg_node(a, (int)gw, b)) return false;
    g = graph_at<T, true>(a, b);
    p = (int)(gw - g.g0);
  } else {
    b = (int)(gw / a.N); p = (int)(gw % a.N);
    g = graph_at<T, false>(a, b);
  }
  return true;
}

// The prologue of the query kernels: the node at cell-order position p of graph g (false: beyond the nodes the graph
// put into its grid), its coordinates xi and its graph's box (bl, binv) or cell (pc).
#define RS_QUERY_ROW()                                                                                                  \
  GraphAt g;                                                                                                            \
  int p;                                                                                                                \
  if (!grid_query_row<T, SEG>(a, gw, g, p)) return;                                                                     \
  const int* cnt = a.cnt + bkt_of<T, SEG>(a, g);                                                                        \
  const int* end = a.end + bkt_of<T, SEG>(a, g);                                                                        \
  if (p >= end[tb_of<T, SEG>(a, g) - 1]) return;                                                                        \
  const size_t g0 = g0_of<T, SEG>(a, g), BN = grid_nodes<T, SEG>(a);                                                    \
  const int i = a.idx[g0 + p];                                                                                          \
  T xi[CD];                                                                                                             \
  _Pragma("unroll") for (int c = 0; c < CD; ++c) xi[c] = a.xs[c * BN + g0 + p];                                         \
  T bl[CD], binv[CD], pc[PBC == PBC_CELL ? CELL_STAGED : 1];                                                            \
  if constexpr (PBC == PBC_CELL) {                                                                                      \
    _Pragma("unroll") for (int t = 0; t < CELL_STAGED; ++t) pc[t] = cell_staged<T>(a.box, lb_of<SEG>(g), CD, t);        \
  } else if constexpr (PBC) {                                                                                           \
    _Pragma("unroll") for (int c = 0; c < CD; ++c) box_axis<T>(a.box, lb_of<SEG>(g), CD, c, bl[c], binv[c]);           \
  }

// The warps per CTA that keep a CTA of SmemLists within RS_WIDE_SMEM (8, or 4 for fp64 at k > 128).
static inline int smem_list_warps(int KP, size_t tbytes) {
  return smem_list_bytes(KP, tbytes) * RS_WARPS <= RS_WIDE_SMEM ? RS_WARPS : RS_WARPS / 2;
}

// The lists of the warp in dynamic shared memory laid out [warps][2 KP] ranks, then [warps][2 KP] indices.
#define RS_SMEM_LIST(sm)                                                                                                \
  T* lk = reinterpret_cast<T*>(sm) + (size_t)warp * 2 * KP;                                                             \
  int* li = reinterpret_cast<int*>(reinterpret_cast<T*>(sm) + (size_t)warps * 2 * KP) + (size_t)warp * 2 * KP;

// k <= 32: the candidate stream, filtered by rank <= r2 and against the current k-th, in a LaneList.
template <typename T, int CD, int PBC, bool SEG = false>
__global__ void __launch_bounds__(RS_WARPS * 32) radius_query_kernel(const RadArgs<T> a) {
  __shared__ T qkey[RS_WARPS][64];
  __shared__ int qidx[RS_WARPS][64];
  __shared__ int sexcl[RS_WARPS][32];
  __shared__ int sdelta[RS_WARPS][32];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const size_t gw = (size_t)blockIdx.x * RS_WARPS + warp;
  if (gw >= grid_nodes<T, SEG>(a)) return;
  RS_QUERY_ROW()
  const int total = row_stream<T, CD, PBC, SEG>(a, g, lane, xi, cnt, end, sexcl[warp], sdelta[warp]);

  LaneList<T> L(qkey[warp], qidx[warp], a.k);
  int nin = 0;                         // this lane's in-radius candidates
  for (int t0 = 0; t0 < total; t0 += 32) {
    const int t = t0 + lane;
    T key = T(INFINITY);
    int j = 0x7fffffff;
    bool pass = false;
    if (t < total) {
      key = stream_rank<T, CD, PBC>(a, g0, BN, t, sexcl[warp], sdelta[warp], xi, bl, binv, pc, j);
      const bool in = key <= a.r2;
      nin += in ? 1 : 0;
      pass = in && L.beats(key, j);
    }
    L.push(pass, key, j, lane);
  }
  L.finish(lane);
  const size_t row = SEG ? (size_t)i : g0 + i;        // the segment form's idx holds node-axis indices
  if (lane < a.k) {
    const size_t o = row * a.k + lane;
    const bool kept = L.bidx != 0x7fffffff;
    a.out_idx[o] = kept ? L.bidx : (a.out_ok ? i : -1);
    if (a.out_ok) a.out_ok[o] = kept ? 1 : 0;
  }
  if (a.out_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nin += __shfl_xor_sync(0xffffffffu, nin, o);
    if (lane == 0) a.out_count[row] = nin;
  }
}

// 32 < k <= RS_WIDE_MAX_K: the candidate stream of radius_query_kernel with the same filter, in a SmemList.
template <typename T, int CD, int PBC, bool SEG = false>
__global__ void __launch_bounds__(RS_WARPS * 32) radius_query_wide_kernel(const RadArgs<T> a, int KP) {
  extern __shared__ __align__(16) unsigned char rsw_sm[];
  __shared__ int sexcl[RS_WARPS][32];
  __shared__ int sdelta[RS_WARPS][32];
  const int warps = blockDim.x / 32, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const size_t gw = (size_t)blockIdx.x * warps + warp;
  if (gw >= grid_nodes<T, SEG>(a)) return;
  RS_QUERY_ROW()
  const int total = row_stream<T, CD, PBC, SEG>(a, g, lane, xi, cnt, end, sexcl[warp], sdelta[warp]);

  RS_SMEM_LIST(rsw_sm)
  SmemList<T> L(lk, li, KP, a.k, lane);
  int nin = 0;                         // this lane's in-radius candidates
  for (int t0 = 0; t0 < total; t0 += 32) {
    const int t = t0 + lane;
    T key = T(INFINITY);
    int j = 0x7fffffff;
    bool pass = false;
    if (t < total) {
      key = stream_rank<T, CD, PBC>(a, g0, BN, t, sexcl[warp], sdelta[warp], xi, bl, binv, pc, j);
      const bool in = key <= a.r2;
      nin += in ? 1 : 0;
      pass = in && L.beats(key, j);
    }
    L.push(pass, key, j, lane);
  }
  L.finish(lane);
  const size_t row = SEG ? (size_t)i : g0 + i;
  for (int s = lane; s < a.k; s += 32) {
    const size_t o = row * a.k + s;
    const bool kept = li[s] != 0x7fffffff;
    a.out_idx[o] = kept ? li[s] : (a.out_ok ? i : -1);
    if (a.out_ok) a.out_ok[o] = kept ? 1 : 0;
  }
  if (a.out_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nin += __shfl_xor_sync(0xffffffffu, nin, o);
    if (lane == 0) a.out_count[row] = nin;
  }
}

// ====================================================================== the kNN grid: k nearest, no cutoff
//
// egnn_knn_select's lists (the same rank, (rank, j) order, 1e5 rank of padded pairs, NaN-last rule and ok bytes) in
// O(N) per graph for C <= 3 and k <= 256.  Seven launches, none synchronising with the host:
//   memsets  bucket counts and the full-scan row count
//   setup    one CTA per graph: extent and count of its insertable nodes -> its KGrid (cell edge, cells per axis)
//   count / scan / scatter   as the radius grid, into the dense cells of the KGrid; padded rows are written here and
//            rows of non-finite nodes listed for the full scan
//   ring     one warp per node in cell order: Chebyshev rings of cells around it until no unvisited node can rank
//            before the k-th; rows the grid cannot decide are listed for the full scan
//   scan     the listed rows against all N nodes of their graph (a SmemList for every k)
constexpr int KG_SETUP_THREADS = 256;
constexpr double KG_FILL = 8.0;            // nodes aimed at per 3^C block of cells, in units of k (DESIGN.md section 6)
constexpr int KG_MAX_RING_CELLS = 4096;    // the largest (2R+1)^C cube of cells a row visits before the full scan
constexpr double KG_MARGIN = 1.0 - 0x1p-10;   // relative rounding margin of the stopping test

struct DMin { __device__ __forceinline__ double operator()(double x, double y) const { return fmin(x, y); } };
struct DMax { __device__ __forceinline__ double operator()(double x, double y) const { return fmax(x, y); } };

// Graph blockIdx.x: the extent lo..hi of its insertable nodes per axis, their count and largest |x|, then its KGrid.
// The cell edge aims at KG_FILL * k nodes per 3^D block of cells, D the number of axes longer than one cell (an axis of
// zero or small extent -- coincident points, a line in 3-D -- gets one cell and leaves the volume), and grows until the
// dense grid fits the Tb buckets.  Periodic axes have their length L (or the cell's perpendicular width) instead of the
// extent and n = max(1, floor(L / cs)) cells of width L / n >= cs, as in the radius grid.
template <typename T, int CD, int PBC, bool SEG = false>
__global__ void __launch_bounds__(KG_SETUP_THREADS) knn_grid_setup_kernel(const RadArgs<T> a) {
  using Red = cub::BlockReduce<double, KG_SETUP_THREADS>;
  __shared__ typename Red::TempStorage tmp;
  __shared__ double res[2 * CD + 2];
  const int b = blockIdx.x;
  if (SEG && !seg_on_grid(a, b)) return;
  const int nodes = SEG ? a.ptr[b + 1] - a.ptr[b] : a.N;
  const int lb = SEG ? 0 : b;                          // the lattice's graph index
  double mn[CD], mx[CD], amax = 0.0, count = 0.0;
#pragma unroll
  for (int c = 0; c < CD; ++c) { mn[c] = INFINITY; mx[c] = -INFINITY; }
  for (int i = threadIdx.x; i < nodes; i += KG_SETUP_THREADS) {
    T x[CD];
    if (!load_node<T, CD>(a, (SEG ? (size_t)a.ptr[b] : (size_t)b * a.N) + i, x)) continue;
    count += 1.0;
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      const double v = (double)x[c];
      mn[c] = fmin(mn[c], v); mx[c] = fmax(mx[c], v); amax = fmax(amax, fabs(v));
    }
  }
#pragma unroll
  for (int c = 0; c < CD; ++c) {
    const double lo = Red(tmp).Reduce(mn[c], DMin());
    __syncthreads();
    const double hi = Red(tmp).Reduce(mx[c], DMax());
    __syncthreads();
    if (threadIdx.x == 0) { res[c] = lo; res[CD + c] = hi; }
  }
  const double am = Red(tmp).Reduce(amax, DMax());
  __syncthreads();
  const double cnt = Red(tmp).Sum(count);
  if (threadIdx.x != 0) return;
  res[2 * CD] = am; res[2 * CD + 1] = cnt;

  KGrid g;
  g.cs = 1.0; g.err = 0.0; g.ok = 0;
  for (int c = 0; c < 3; ++c) {
    g.lo[c] = 0.0; g.L[c] = 0.0; g.w[c] = 1.0; g.n[c] = 1;
    for (int d = 0; d < 3; ++d) g.G[c][d] = 0.0;
  }
  const double ins = res[2 * CD + 1];
  double len[CD];
  bool per[CD];
  if constexpr (PBC == PBC_CELL) {
    double G[CD][CD];
    cell_inverse<T, CD>(a.box + (size_t)lb * CD * CD, G, per);
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      double g2 = 0.0;
#pragma unroll
      for (int d = c; d < CD; ++d) g2 = fma(G[d][c], G[d][c], g2);
      len[c] = per[c] ? 1.0 / sqrt(g2) : res[CD + c] - res[c];
#pragma unroll
      for (int d = 0; d < CD; ++d) g.G[c][d] = G[c][d];
    }
  } else {
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      const T l = PBC == PBC_BOX ? a.box[(size_t)lb * CD + c] : T(0);
      per[c] = l > T(0) && l < T(INFINITY);
      len[c] = per[c] ? (double)l : res[CD + c] - res[c];
    }
  }
  bool usable = ins >= (double)a.k;
#pragma unroll
  for (int c = 0; c < CD; ++c) usable = usable && len[c] >= 0.0 && len[c] < INFINITY;
  if (usable) {
    // the cell edge over the axes longer than it, recomputed as short axes drop out
    bool act[CD];
#pragma unroll
    for (int c = 0; c < CD; ++c) act[c] = len[c] > 0.0;
    double cs = 1.0;
    for (int it = 0; it < CD; ++it) {
      int D = 0;
      double V = 1.0, blk = 1.0;
      for (int c = 0; c < CD; ++c) if (act[c]) { ++D; V *= len[c]; blk *= 3.0; }
      if (D == 0) break;
      cs = pow(KG_FILL * a.k * V / (blk * ins), 1.0 / D);
      bool dropped = false;
      for (int c = 0; c < CD; ++c) if (act[c] && len[c] < cs) { act[c] = false; dropped = true; }
      if (!dropped) break;
    }
    usable = cs > 0.0 && cs < INFINITY;
    for (int grow = 0; usable; ++grow) {             // the dense grid must fit the Tb buckets
      double cells = 1.0;
      for (int c = 0; c < CD; ++c) {
        const double q = floor(len[c] / cs);
        cells *= per[c] ? fmax(q, 1.0) : q + 1.0;
      }
      if (cells <= (double)(SEG ? rs_buckets(nodes) : a.Tb)) break;
      cs *= 2.0;
      usable = grow < 2100;
    }
    if (usable) {
      g.cs = cs;
      g.ok = 1;
      for (int c = 0; c < CD; ++c) {
        const double q = floor(len[c] / cs);
        g.n[c] = per[c] ? (int)fmax(q, 1.0) : (int)q + 1;
        g.lo[c] = per[c] ? 0.0 : res[c];
        g.L[c] = per[c] ? (PBC == PBC_CELL ? 1.0 : len[c]) : 0.0;
        g.w[c] = per[c] ? len[c] / g.n[c] : cs;
      }
      // Rounding allowance (DESIGN.md section 5): binning in double moves a cell face by at most a few ulp of the
      // coordinates, and under a box or cell the wrapped pair vector carries the rounding of the unwrapped difference,
      // u |x_i - x_j| per step, with |x_i - x_j| <= 2 max |x|.
      const double u = sizeof(T) == 4 ? 0x1p-24 : 0x1p-53;
      const double am2 = 2.0 * CD * res[2 * CD];
      g.err = 0x1p-40 * am2 + (PBC != PBC_NONE ? 16.0 * u * am2 : 0.0);
    }
  }
  if (!usable) {                                       // every node into cell 0; the ring kernel lists every row
    g.ok = 0;
    for (int c = 0; c < 3; ++c) { g.n[c] = 1; g.L[c] = 0.0; g.lo[c] = 0.0; }
    g.cs = 1.0;
  }
  a.kg[b] = g;
}

// Row of node i (b, cell-order position p): the rings of cells around its cell, R = 0, 1, ..., each read as streams
// of up to 32 cells (bucket_stream) whose nodes are offered to the list L.  Offsets along a periodic axis of n cells
// are taken in [-(n-1)/2, n-1-(n-1)/2], so every cell is visited once; along an aperiodic axis they are clipped to the
// graph's cells.  After ring R an unvisited node is at least R w_c away along some axis c whose cells are not all
// visited, so once the k-th (rank, j) ranks below that distance squared, with the rounding margin, no unvisited pair
// can rank before or tie with it.  Returns false when the row is left to the full scan: no usable grid, the ring
// budget exhausted, or a k-th rank that is not finite or (under a mask) reaches the padded pairs' 1e5.
template <typename T, int CD, int PBC, class List>
__device__ __forceinline__ bool knn_ring_row(const RadArgs<T>& a, List& L, const GraphAt& ga, int lane, const T (&xi)[CD],
                                             const T (&bl)[CD], const T (&binv)[CD], const T* pc, const int* cnt,
                                             const int* end, size_t g0, size_t BN, int* wexcl, int* wdelta) {
  const KGrid& g = a.kg[ga.b];
  if (!g.ok) return false;
  int cc[CD], dlo[CD], dhi[CD], n[CD];
  knn_cell<T, CD, PBC>(g, xi, cc);
#pragma unroll
  for (int c = 0; c < CD; ++c) {
    n[c] = g.n[c];
    dlo[c] = g.L[c] > 0.0 ? -((n[c] - 1) / 2) : -cc[c];
    dhi[c] = g.L[c] > 0.0 ? n[c] - 1 - (n[c] - 1) / 2 : n[c] - 1 - cc[c];
  }
  for (int R = 0;; ++R) {
    const int side = 2 * R + 1;
    int ncube = 1;
#pragma unroll
    for (int c = 0; c < CD; ++c) ncube *= side;
    for (int u0 = 0; u0 < ncube; u0 += 32) {
      const int u = u0 + lane;
      int cell = -1;
      if (u < ncube) {
        int r = u, t = 0, mul = 1;
        bool in = true, ring = false;
#pragma unroll
        for (int c = 0; c < CD; ++c) {
          const int d = r % side - R;
          r /= side;
          in = in && d >= dlo[c] && d <= dhi[c];
          ring = ring || d == R || d == -R;
          int v = cc[c] + d;
          v = v < 0 ? v + n[c] : (v >= n[c] ? v - n[c] : v);
          t += v * mul;
          mul *= n[c];
        }
        if (in && ring) cell = t;
      }
      __syncwarp();                                    // the previous stream has been read
      const int total = bucket_stream(lane, cell >= 0, cell, cnt, end, wexcl, wdelta);
      for (int t0 = 0; t0 < total; t0 += 32) {
        const int t = t0 + lane;
        T key = T(INFINITY);
        int j = 0x7fffffff;
        bool pass = false;
        if (t < total) {
          key = stream_rank<T, CD, PBC>(a, g0, BN, t, wexcl, wdelta, xi, bl, binv, pc, j);
          pass = L.beats(key, j);
        }
        L.push(pass, key, j, lane);
      }
    }
    L.finish(lane);
    L.refresh();                                       // thr_key / thr_idx: the k-th of every pair offered so far
    bool covered = true;
    double w = INFINITY;
#pragma unroll
    for (int c = 0; c < CD; ++c)
      if (dlo[c] < -R || dhi[c] > R) { covered = false; w = fmin(w, g.w[c]); }
    if (covered) break;
    const T thr = L.thr_key;
    if (L.thr_idx != 0x7fffffff) {
      const double bd = R * w * KG_MARGIN - g.err;
      if (bd > 0.0 && bd * bd >= 0x1p-96 && (double)thr < bd * bd * KG_MARGIN) break;
    }
    int next = 1;
#pragma unroll
    for (int c = 0; c < CD; ++c) next *= side + 2;
    if (next > KG_MAX_RING_CELLS) return false;
  }
  const T thr = L.thr_key;
  return thr < T(INFINITY) && !(a.mask && thr >= T(1e5));
}

// The ring query: one warp per node in cell order; k <= 32 in a LaneList, larger k in a SmemList (KP > 0).
template <typename T, int CD, int PBC, bool WIDE, bool SEG = false>
__global__ void __launch_bounds__(RS_WARPS * 32) knn_ring_kernel(const RadArgs<T> a, int KP) {
  extern __shared__ __align__(16) unsigned char kgr_sm[];
  __shared__ T qkey[WIDE ? 1 : RS_WARPS][64];
  __shared__ int qidx[WIDE ? 1 : RS_WARPS][64];
  __shared__ int sexcl[RS_WARPS][32];
  __shared__ int sdelta[RS_WARPS][32];
  const int warps = blockDim.x / 32, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const size_t gw = (size_t)blockIdx.x * warps + warp;
  if (gw >= grid_nodes<T, SEG>(a)) return;
  RS_QUERY_ROW()
  const size_t row = SEG ? (size_t)i : g0 + i;
  if constexpr (WIDE) {
    RS_SMEM_LIST(kgr_sm)
    SmemList<T> L(lk, li, KP, a.k, lane);
    if (!knn_ring_row<T, CD, PBC>(a, L, g, lane, xi, bl, binv, pc, cnt, end, g0, BN, sexcl[warp], sdelta[warp])) {
      if (lane == 0) a.fb_rows[atomicAdd(a.fb_count, 1)] = (int)row;
      return;
    }
    for (int s = lane; s < a.k; s += 32) {
      a.out_idx[row * a.k + s] = li[s];
      if (a.out_ok) a.out_ok[row * a.k + s] = lk[s] <= a.vr ? 1 : 0;
    }
  } else {
    LaneList<T> L(qkey[warp], qidx[warp], a.k);
    if (!knn_ring_row<T, CD, PBC>(a, L, g, lane, xi, bl, binv, pc, cnt, end, g0, BN, sexcl[warp], sdelta[warp])) {
      if (lane == 0) a.fb_rows[atomicAdd(a.fb_count, 1)] = (int)row;
      return;
    }
    if (lane < a.k) {
      a.out_idx[row * a.k + lane] = L.bidx;
      if (a.out_ok) a.out_ok[row * a.k + lane] = L.bkey <= a.vr ? 1 : 0;
    }
  }
}

// The listed rows, each against all N nodes of its graph with egnn_knn_select's rank: 1e5 to a padded node, and a NaN
// rank ordered as (+inf, j + N), after every +inf and by index, written as j with ok = 0 (knn_block_sort_kernel's
// rule).  Grid-stride over the list, whose length only the device knows.  In the segment form a row is ranked against
// the n_b nodes of its own graph, j on the node axis and N = T.
template <typename T, int CD, int PBC, bool SEG = false>
__global__ void __launch_bounds__(RS_WARPS * 32) knn_scan_kernel(const RadArgs<T> a, int KP) {
  extern __shared__ __align__(16) unsigned char kgs_sm[];
  const int warps = blockDim.x / 32, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  RS_SMEM_LIST(kgs_sm)
  const int rows = *a.fb_count;
  for (int r = blockIdx.x * warps + warp; r < rows; r += gridDim.x * warps) {
    const size_t row = (size_t)a.fb_rows[r];
    int b = (int)(row / a.N), nj = a.N;
    if constexpr (SEG) {
      seg_node(a, (int)row, b);                        // listed rows are on the grid
      nj = a.ptr[b + 1] - a.ptr[b];
    }
    const GraphAt ga = graph_at<T, SEG>(a, b);
    const size_t g0 = g0_of<T, SEG>(a, ga);
    const int j0 = SEG ? (int)g0 : 0;                  // the node index of candidate 0
    T xi[CD];
#pragma unroll
    for (int c = 0; c < CD; ++c) xi[c] = a.coors[row * CD + c];
    T bl[CD], binv[CD], pc[PBC == PBC_CELL ? CELL_STAGED : 1];
    if constexpr (PBC == PBC_CELL) {
#pragma unroll
      for (int t = 0; t < CELL_STAGED; ++t) pc[t] = cell_staged<T>(a.box, lb_of<SEG>(ga), CD, t);
    } else if constexpr (PBC) {
#pragma unroll
      for (int c = 0; c < CD; ++c) box_axis<T>(a.box, lb_of<SEG>(ga), CD, c, bl[c], binv[c]);
    }
    SmemList<T> L(lk, li, KP, a.k, lane);
    for (int jb = 0; jb < nj; jb += 32) {
      const int j = jb + lane;
      T key = T(INFINITY);
      int jk = 0x7fffffff;
      bool pass = false;
      if (j < nj) {
        const T* xj = a.coors + (g0 + j) * CD;
        key = pair_rank<T, CD, PBC>(xi, [&](int c) { return xj[c]; }, CD, bl, binv, pc);
        if (a.mask && !a.mask[g0 + j]) key = T(1e5);
        jk = j0 + j;
        if (key != key) { key = T(INFINITY); jk = j0 + j + a.N; }
        pass = L.beats(key, jk);
      }
      L.push(pass, key, jk, lane);
    }
    L.finish(lane);
    for (int s = lane; s < a.k; s += 32) {
      const bool nan_rank = li[s] >= a.N;
      a.out_idx[row * a.k + s] = nan_rank ? li[s] - a.N : li[s];
      if (a.out_ok) a.out_ok[row * a.k + s] = !nan_rank && lk[s] <= a.vr ? 1 : 0;
    }
    __syncwarp();
  }
}

// ====================================================================== host side of both grids

// One select on the radius grid (GRID_RADIUS) or the kNN grid (GRID_KNN): one memset of the bucket counts, then count /
// scan / scatter into the grid's buckets and the query, one warp per row: radius_query_kernel; or, on the kNN grid,
// knn_grid_setup_kernel first, then knn_ring_kernel and knn_scan_kernel for the rows it leaves.  The segment form (SEG)
// launches the same sequence over the T nodes and G graphs of a packed batch; graphs off the grid exit at once.
template <typename T, int CD, int PBC, int GRID, bool SEG = false>
static int launch_grid(const RadArgs<T>& a, cudaStream_t st) {
  const size_t nodes = SEG ? (size_t)a.N : (size_t)a.B * a.N;
  const unsigned gn = (unsigned)((nodes + RS_THREADS - 1) / RS_THREADS);
  EGNN_CUDA_TRY(cudaMemsetAsync(a.cnt, 0, (SEG ? 4 * nodes : (size_t)a.B * a.Tb) * sizeof(int), st));
  if constexpr (GRID == GRID_KNN) {
    EGNN_CUDA_TRY(cudaMemsetAsync(a.fb_count, 0, sizeof(int), st));
    knn_grid_setup_kernel<T, CD, PBC, SEG><<<a.B, KG_SETUP_THREADS, 0, st>>>(a);
    EGNN_LAUNCH_CHECK();
  }
  radius_count_kernel<T, CD, PBC, GRID, SEG><<<gn, RS_THREADS, 0, st>>>(a);
  EGNN_LAUNCH_CHECK();
  if constexpr (SEG) radius_scan_seg_kernel<T><<<a.B, RS_SCAN_THREADS, 0, st>>>(a);
  else radius_scan_kernel<<<a.B, RS_SCAN_THREADS, 0, st>>>(a.cnt, a.end, a.Tb);
  EGNN_LAUNCH_CHECK();
  radius_scatter_kernel<T, CD, PBC, GRID, SEG><<<gn, RS_THREADS, 0, st>>>(a);
  EGNN_LAUNCH_CHECK();
  // k <= 32: RS_WARPS rows per CTA, lists in lanes; larger k: SmemLists in dynamic shared memory
  const int KP = list_kp(a.k), warps = smem_list_warps(KP, sizeof(T));
  const size_t smem = warps * smem_list_bytes(KP, sizeof(T));
  const unsigned rows = (unsigned)((nodes + RS_WARPS - 1) / RS_WARPS), wide_rows = (unsigned)((nodes + warps - 1) / warps);
  if constexpr (GRID == GRID_KNN) {
    if (a.k <= 32) knn_ring_kernel<T, CD, PBC, false, SEG><<<rows, RS_WARPS * 32, 0, st>>>(a, 0);
    else knn_ring_kernel<T, CD, PBC, true, SEG><<<wide_rows, warps * 32, smem, st>>>(a, KP);
    EGNN_LAUNCH_CHECK();
    int sms = 0;
    EGNN_TRY(sm_count(&sms));
    knn_scan_kernel<T, CD, PBC, SEG><<<(wide_rows < 4u * sms ? wide_rows : 4u * sms), warps * 32, smem, st>>>(a, KP);
    EGNN_LAUNCH_CHECK();
    count_launch(6);
  } else {
    if (a.k <= 32) radius_query_kernel<T, CD, PBC, SEG><<<rows, RS_WARPS * 32, 0, st>>>(a);
    else radius_query_wide_kernel<T, CD, PBC, SEG><<<wide_rows, warps * 32, smem, st>>>(a, KP);
    EGNN_LAUNCH_CHECK();
    count_launch(4);
  }
  return EGNN_OK;
}

// The C x lattice instantiation of launch_grid.
template <typename T, int GRID, bool SEG>
static int grid_dispatch(const RadArgs<T>& a, int C, const void* box, int pbc, cudaStream_t st) {
  if (box && pbc == PBC_CELL) {
    if (C == 2) return launch_grid<T, 2, PBC_CELL, GRID, SEG>(a, st);
    if (C == 3) return launch_grid<T, 3, PBC_CELL, GRID, SEG>(a, st);
    return EGNN_ERR_SHAPE;
  }
  switch (C * 2 + (box ? 1 : 0)) {
    case 2: return launch_grid<T, 1, PBC_NONE, GRID, SEG>(a, st);
    case 3: return launch_grid<T, 1, PBC_BOX, GRID, SEG>(a, st);
    case 4: return launch_grid<T, 2, PBC_NONE, GRID, SEG>(a, st);
    case 5: return launch_grid<T, 2, PBC_BOX, GRID, SEG>(a, st);
    case 6: return launch_grid<T, 3, PBC_NONE, GRID, SEG>(a, st);
    case 7: return launch_grid<T, 3, PBC_BOX, GRID, SEG>(a, st);
    default: return EGNN_ERR_UNSUPPORTED;
  }
}

// r: the squared radius (GRID_RADIUS) or valid_radius (GRID_KNN) as the caller passes it; the kernels compare in T.
// box: null, a [B,C] box, or a [B,C,C] cell under pbc = PBC_CELL.
// The segment form (seg non-null: B = G graphs, N = T nodes): seg->ptr, seg->seg_valid and seg->min_n are taken over,
// and the scratch is laid out for T nodes in 4 T buckets.
template <typename T, int GRID>
static int grid_select(int B, int N, int C, int k, const void* coors, const uint8_t* mask, const void* box, double r,
                       int32_t* out_idx, uint8_t* out_ok, int32_t* out_count, void* ws, cudaStream_t st, int pbc,
                       const RadArgs<T>* seg = nullptr) {
  const KnnWs L = seg ? knn_ws_layout(B, (size_t)N, 4 * (size_t)N, C, sizeof(T))
                      : knn_ws_layout(B, (size_t)B * N, (size_t)B * rs_buckets(N), C, sizeof(T));   // radius: the cell part
  char* base = static_cast<char*>(ws);
  RadArgs<T> a{};
  a.B = B; a.N = N; a.k = k; a.Tb = seg ? 0 : rs_buckets(N);
  if (seg) { a.ptr = seg->ptr; a.seg_valid = seg->seg_valid; a.min_n = seg->min_n; }
  a.coors = static_cast<const T*>(coors); a.mask = mask; a.box = static_cast<const T*>(box);
  a.cnt = reinterpret_cast<int*>(base + L.cell.cnt);
  a.end = reinterpret_cast<int*>(base + L.cell.end);
  a.xs = reinterpret_cast<T*>(base + L.cell.xs);
  a.idx = reinterpret_cast<int*>(base + L.cell.idx);
  a.out_idx = out_idx; a.out_ok = out_ok; a.out_count = out_count;
  if constexpr (GRID == GRID_KNN) {
    a.vr = (T)r;
    a.kg = reinterpret_cast<KGrid*>(base + L.kg);
    a.fb_rows = reinterpret_cast<int*>(base + L.fb);
    a.fb_count = reinterpret_cast<int*>(base + L.nfb);
  } else {
    a.r2 = (T)r;
    a.cs = sqrt((double)a.r2) * (1.0 + 0x1p-10);
  }
  return seg ? grid_dispatch<T, GRID, true>(a, C, box, pbc, st) : grid_dispatch<T, GRID, false>(a, C, box, pbc, st);
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
    return grid_select<double, GRID_RADIUS>(B, N, C, k, coors, mask, box, r2, out_idx, out_ok, out_count, ws, st, pbc);
  }
  if (dtype != EGNN_DTYPE_F32) return EGNN_ERR_UNSUPPORTED;
  if (!((float)r2 > 0.f)) return EGNN_ERR_SHAPE;
  return grid_select<float, GRID_RADIUS>(B, N, C, k, coors, mask, box, r2, out_idx, out_ok, out_count, ws, st, pbc);
}

// Smallest N per graph at which a flagged layer selects on the kNN grid (DESIGN.md section 6).
// EGNN_B200_KNN_GRID_MIN_N overrides it at every call (0 = always, a huge value = never).
constexpr long KNN_GRID_MIN_N = 8192;
static long knn_grid_min_n() {
  const char* e = getenv("EGNN_B200_KNN_GRID_MIN_N");
  return e ? strtol(e, nullptr, 10) : KNN_GRID_MIN_N;
}

bool knn_grid_runs(const EgnnLayerDesc& d, const EgnnLayerIO& io) {
  return !io.adj && !io.nbr_idx && knn_grid_eligible(d) && !cell_select_runs(d, io) && d.N >= knn_grid_min_n();
}

int knn_grid_dispatch(int32_t dtype, int B, int N, int C, int k, const void* coors, const uint8_t* mask, const void* box,
                      double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* ws, cudaStream_t st, int pbc) {
  if (!coors || !out_idx || !ws) return EGNN_ERR_NULL;
  EGNN_TRY(radius_check(B, N, C, k, RS_WIDE_MAX_K));
  if (dtype == EGNN_DTYPE_F64)
    return grid_select<double, GRID_KNN>(B, N, C, k, coors, mask, box, valid_radius, out_idx, out_ok, nullptr, ws, st,
                                         pbc);
  if (dtype != EGNN_DTYPE_F32) return EGNN_ERR_UNSUPPORTED;
  return grid_select<float, GRID_KNN>(B, N, C, k, coors, mask, box, valid_radius, out_idx, out_ok, nullptr, ws, st, pbc);
}

// ---------------------------------------------------------------- packed batches (segment_select.cu's grid entries)

size_t packed_grid_ws_bytes(bool knn, int G, int T, int C) {
  const KnnWs w = knn_ws_layout(G, (size_t)T, 4 * (size_t)T, C, 8);
  return knn ? w.total : w.cell.total;
}

// The smallest graph a packed select puts on the grid: the unpacked threshold, read now, and at least k; INT_MAX when
// this call puts none there (the radius grid with r outside (0, 1e5) in the coordinates' type, as cell_select_eligible).
int packed_grid_min_n(bool knn, int32_t dtype, int k, double r) {
  if (!knn) {
    const double r2 = dtype == EGNN_DTYPE_F64 ? r : (double)(float)r;
    if (!(r2 > 0.0 && r2 < 1e5)) return INT_MAX;
  }
  const long thr = knn ? knn_grid_min_n() : cell_select_min_n();
  const long m = thr > k ? thr : k;
  return m > INT_MAX ? INT_MAX : (int)m;
}

int packed_grid_launch(bool knn, int32_t dtype, int G, int T, int C, int k, int min_n, const int32_t* ptr,
                       const int* seg_valid, const void* coors, const uint8_t* mask, const void* lattice, int pbc,
                       double r, int32_t* out_idx, uint8_t* out_ok, void* ws, cudaStream_t st) {
  if (dtype == EGNN_DTYPE_F64) {
    RadArgs<double> s{};
    s.ptr = ptr; s.seg_valid = seg_valid; s.min_n = min_n;
    return knn ? grid_select<double, GRID_KNN>(G, T, C, k, coors, mask, lattice, r, out_idx, out_ok, nullptr, ws, st, pbc, &s)
               : grid_select<double, GRID_RADIUS>(G, T, C, k, coors, mask, lattice, r, out_idx, out_ok, nullptr, ws, st,
                                                  pbc, &s);
  }
  RadArgs<float> s{};
  s.ptr = ptr; s.seg_valid = seg_valid; s.min_n = min_n;
  return knn ? grid_select<float, GRID_KNN>(G, T, C, k, coors, mask, lattice, r, out_idx, out_ok, nullptr, ws, st, pbc, &s)
             : grid_select<float, GRID_RADIUS>(G, T, C, k, coors, mask, lattice, r, out_idx, out_ok, nullptr, ws, st, pbc,
                                               &s);
}

// The public entries: egnn_radius_select* with k <= 32, egnn_radius_select_wide* and egnn_knn_grid_select* with
// k <= RS_WIDE_MAX_K.  Workspace sizes are for float64 coordinates, which covers both types.
static int grid_ws_entry(int grid, int max_k, int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes) {
  if (!out_bytes) return EGNN_ERR_NULL;
  EGNN_TRY(radius_check(B, N, C, k, max_k));
  *out_bytes = grid_ws_bytes(grid, B, N, C, 8);
  return EGNN_OK;
}

// The checks of a public select entry before the select's own.  lattice: a [B,C] box (pbc = PBC_BOX, may be null) or
// a [B,C,C] cell (PBC_CELL).
static int grid_entry_check(int grid, int max_k, int pbc, int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k,
                            const void* lattice, void* workspace, size_t workspace_bytes) {
  if (!workspace || (pbc == PBC_CELL && !lattice)) return EGNN_ERR_NULL;
  if (pbc == PBC_CELL && (C < 2 || C > 3)) return EGNN_ERR_SHAPE;    // a cell is 2-D or 3-D (before radius_check's C > 3)
  EGNN_TRY(radius_check(B, N, C, k, max_k));
  if ((uintptr_t)workspace & 0xFF) return EGNN_ERR_ALIGN;
  if (workspace_bytes < grid_ws_bytes(grid, B, N, C, dtype == EGNN_DTYPE_F64 ? 8 : 4)) return EGNN_ERR_WORKSPACE;
  return EGNN_OK;
}

static int radius_entry(int max_k, int pbc, int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                        const uint8_t* mask, const void* lattice, double r2, int32_t* out_idx, int32_t* out_count,
                        void* workspace, size_t workspace_bytes, void* stream) {
  EGNN_TRY(grid_entry_check(GRID_RADIUS, max_k, pbc, dtype, B, N, C, k, lattice, workspace, workspace_bytes));
  return cell_select_dispatch(dtype, B, N, C, k, coors, mask, lattice, r2, out_idx, nullptr, out_count, workspace,
                              static_cast<cudaStream_t>(stream), pbc);
}

static int knn_entry(int pbc, int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                     const uint8_t* mask, const void* lattice, double valid_radius, int32_t* out_idx, uint8_t* out_ok,
                     void* workspace, size_t workspace_bytes, void* stream) {
  EGNN_TRY(grid_entry_check(GRID_KNN, RS_WIDE_MAX_K, pbc, dtype, B, N, C, k, lattice, workspace, workspace_bytes));
  return knn_grid_dispatch(dtype, B, N, C, k, coors, mask, lattice, valid_radius, out_idx, out_ok, workspace,
                           static_cast<cudaStream_t>(stream), pbc);
}

}  // namespace egnn

extern "C" int egnn_radius_select_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes) {
  return egnn::grid_ws_entry(egnn::GRID_RADIUS, 32, B, N, C, k, out_bytes);
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
  return egnn::grid_ws_entry(egnn::GRID_RADIUS, egnn::RS_WIDE_MAX_K, B, N, C, k, out_bytes);
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

extern "C" int egnn_knn_grid_select_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes) {
  return egnn::grid_ws_entry(egnn::GRID_KNN, egnn::RS_WIDE_MAX_K, B, N, C, k, out_bytes);
}

extern "C" int egnn_knn_grid_select(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                    const uint8_t* mask, const void* box, double valid_radius, int32_t* out_idx,
                                    uint8_t* out_ok, void* workspace, size_t workspace_bytes, void* stream) {
  return egnn::knn_entry(egnn::PBC_BOX, dtype, B, N, C, k, coors, mask, box, valid_radius, out_idx, out_ok, workspace,
                         workspace_bytes, stream);
}

extern "C" int egnn_knn_grid_select_triclinic(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k,
                                              const void* coors, const uint8_t* mask, const void* cell,
                                              double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                              size_t workspace_bytes, void* stream) {
  return egnn::knn_entry(egnn::PBC_CELL, dtype, B, N, C, k, coors, mask, cell, valid_radius, out_idx, out_ok, workspace,
                         workspace_bytes, stream);
}

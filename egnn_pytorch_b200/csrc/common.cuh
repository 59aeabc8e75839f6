// Shared helpers for libegnn_b200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stddef.h>
#include <math.h>
#include <map>
#include <mutex>
#include <utility>

#include "../../include/egnn_b200.h"

namespace egnn {

// ------------------------------------------------------------------ error plumbing
#define EGNN_CUDA_TRY(expr)                                         \
  do {                                                              \
    cudaError_t _e = (expr);                                        \
    if (_e != cudaSuccess) return EGNN_ERR_CUDA - (int)_e;          \
  } while (0)

#define EGNN_TRY(expr)                                              \
  do {                                                              \
    int _r = (expr);                                                \
    if (_r != EGNN_OK) return _r;                                   \
  } while (0)

// Launch check that does not synchronise: catches bad configurations at enqueue time.
#define EGNN_LAUNCH_CHECK() EGNN_CUDA_TRY(cudaPeekAtLastError())

// Opt `kernel` in to `bytes` of dynamic shared memory on the current device.  One process-wide table remembers what
// each (device, kernel) was raised to, so the attribute is set once per new maximum, never lowered (one kernel is
// launched from several translation units with different needs), and a launch that needs no more costs no API call
// beyond cudaGetDevice.
inline int ensure_dynamic_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return EGNN_OK;
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> raised;
  int dev = 0;
  EGNN_CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = raised[{dev, kernel}];
  if (cur < bytes) {
    EGNN_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    cur = bytes;
  }
  return EGNN_OK;
}
template <typename... A>
inline int ensure_dynamic_smem(void (*kernel)(A...), size_t bytes) {
  return ensure_dynamic_smem(reinterpret_cast<const void*>(kernel), bytes);
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline size_t round_up(size_t a, size_t b) { return (a + b - 1) / b * b; }
__host__ __device__ inline int round_up_i(int a, int b) { return (a + b - 1) / b * b; }

// Streaming-multiprocessor count of the current device (cached per device): grid sizes follow the GPU they run on.
inline int sm_count(int* out) {
  static std::mutex mu;
  static int cached[64] = {0};
  int dev = 0;
  EGNN_CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (dev < 64 && cached[dev] > 0) { *out = cached[dev]; return EGNN_OK; }
  int n = 0;
  EGNN_CUDA_TRY(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  if (dev < 64) cached[dev] = n;
  *out = n;
  return EGNN_OK;
}

// Neighbour lists of a layer with k > 0 (egnn_pytorch.py:237-260), ranked into *nbr_idx / *nbr_ok (workspace arrays
// of [B,N,k]); in edge-list mode (io.nbr_idx set) the pointers are redirected to the caller's lists and *nbr_ok to null.
// box: [B,C] periodic box lengths (pbc = PBC_BOX) or a [B,C,C] lower-triangular cell (pbc = PBC_CELL) in the
// coordinates' type, distances then being those of the wrapped pair vector; null with PBC_NONE.
// cell_ws: the layer's cell-grid scratch (cell_select_layer_ws_bytes(d) bytes), or null when it has none.
int select_neighbors(const EgnnLayerDesc& d, const EgnnLayerIO& io, int32_t** nbr_idx, uint8_t** nbr_ok, cudaStream_t st,
                     const void* box = nullptr, void* cell_ws = nullptr, int pbc = 0);

// The cell-grid radius select (radius_select.cu).  A layer is eligible from its descriptor alone (1 <= k <= 32, or <= 256
// under EGNN_FLAG_CELL_SELECT_WIDE, C <= 3, 0 < (T)valid_radius < 1e5, no only_sparse / batched adjacency / per-slot edges); its forward workspace then carries
// cell_select_layer_ws_bytes(d) bytes of scratch (0 for a layer that neither grid may serve; the kNN grid's, which
// contains the radius grid's, under EGNN_FLAG_KNN_GRID), whatever the size thresholds.
// cell_select_runs adds what the call decides: a mask, no adjacency, no caller lists and N >= the threshold.
bool cell_select_eligible(const EgnnLayerDesc& d);
size_t cell_select_layer_ws_bytes(const EgnnLayerDesc& d);
bool cell_select_runs(const EgnnLayerDesc& d, const EgnnLayerIO& io);
int cell_select_dispatch(int32_t dtype, int B, int N, int C, int k, const void* coors, const uint8_t* mask,
                         const void* box, double r2, int32_t* out_idx, uint8_t* out_ok, int32_t* out_count, void* ws,
                         cudaStream_t st, int pbc);
// The kNN grid (radius_select.cu): under EGNN_FLAG_KNN_GRID a layer is eligible from its descriptor alone (1 <= k <= 32,
// or <= 256 under EGNN_FLAG_CELL_SELECT_WIDE, C <= 3, no only_sparse / batched adjacency / per-slot edges), and its
// workspace then ends in the kNN grid's scratch (cell_select_layer_ws_bytes).  knn_grid_runs adds what the call decides:
// the radius grid does not run, no adjacency, no caller lists and N >= the threshold.
bool knn_grid_runs(const EgnnLayerDesc& d, const EgnnLayerIO& io);
int knn_grid_dispatch(int32_t dtype, int B, int N, int C, int k, const void* coors, const uint8_t* mask, const void* box,
                      double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* ws, cudaStream_t st, int pbc);
// Either grid on a packed batch (radius_select.cu, for segment_select.cu's grid entries; knn: the kNN grid, else the
// radius grid): its scratch for T nodes of G graphs (either coordinate type), the smallest graph this call puts on it
// (INT_MAX: none), and its launches for the graphs of at least min_n nodes while *seg_valid (set on the device).
size_t packed_grid_ws_bytes(bool knn, int G, int T, int C);
int packed_grid_min_n(bool knn, int32_t dtype, int k, double r);
int packed_grid_launch(bool knn, int32_t dtype, int G, int T, int C, int k, int min_n, const int32_t* ptr,
                       const int* seg_valid, const void* coors, const uint8_t* mask, const void* lattice, int pbc,
                       double r, int32_t* out_idx, uint8_t* out_ok, void* ws, cudaStream_t st);

// ------------------------------------------------------------------ derived sizes
struct Dims {
  int B, N, C, dim, edge_dim, label_dim, num_labels, m, F, k;
  int Qd;      // distance feature channels 2F+1            (egnn_pytorch.py:34-41)
  int Q;       // per-pair scalar channels Qd + edge_dim
  int E;       // edge_input_dim                             (egnn_pytorch.py:175)
  int H;       // hidden width 2E                            (egnn_pytorch.py:179)
  int Hp;      // H rounded up to 8 (zero padded)
  int M;       // B*N rows
  int row0, row1;
};

inline Dims make_dims(const EgnnLayerDesc& d) {
  Dims s;
  s.B = d.B; s.N = d.N; s.C = d.C; s.dim = d.dim; s.edge_dim = d.edge_dim;
  s.label_dim = d.label_dim; s.num_labels = d.num_labels; s.m = d.m_dim; s.F = d.fourier; s.k = d.k;
  s.Qd = 2 * d.fourier + 1;
  s.Q = s.Qd + d.edge_dim;
  s.E = 2 * d.dim + s.Q + d.label_dim;
  s.H = 2 * s.E;
  s.Hp = round_up_i(s.H, 8);
  s.M = d.B * d.N;
  s.row0 = d.row_begin; s.row1 = d.row_end;
  if (s.row0 == 0 && s.row1 == 0) s.row1 = d.N;
  return s;
}

// Row blocks (EGNN_FLAG_ROW_PARTIAL_GRADS with a range other than all rows): the per-pair buffers (pre2, the backward
// record) hold the block's rows only, B x (row1 - row0), row i at i - row0.  The pair kernels take this as a template
// parameter BLK, so the instantiations without a row block keep the plain node-order arithmetic and their arguments.
inline bool row_block(const Dims& s, uint32_t flags) {
  return (flags & EGNN_FLAG_ROW_PARTIAL_GRADS) && (s.row0 != 0 || s.row1 != s.N);
}
// Rows per graph of the per-pair buffers.
inline int pair_rows(const Dims& s, uint32_t flags) { return row_block(s, flags) ? s.row1 - s.row0 : s.N; }
// Row of node (b, i) in the per-pair buffers.
template <bool BLK>
__host__ __device__ __forceinline__ size_t pair_row(const Dims& s, int b, int i) {
  return BLK ? (size_t)b * (s.row1 - s.row0) + (i - s.row0) : (size_t)b * s.N + i;
}

// The edge-feature row of slot `slot` of row node_i = b*N + i, whose neighbour is j: [B,N,k,edge_dim] per slot under
// EGNN_FLAG_EDGES_PER_SLOT, else [B,N,N,edge_dim] per pair.  Every reader and the per-slot gradient store use this one
// rule.  A slot beyond k (a padding lane) reads slot 0, which always exists.
template <typename E>
__device__ __forceinline__ E* edge_row(E* edges, bool per_slot, size_t node_i, int slot, int j, int N, int k, int edge_dim) {
  const size_t r = per_slot ? node_i * k + (slot < k ? slot : 0) : node_i * N + j;
  return edges + r * edge_dim;
}

// ------------------------------------------------------------------ dropout (training mode, egnn_pytorch.py:176-208)
// nn.Dropout(p) sits between Linear-1 and SiLU of edge_mlp / node_mlp / coors_mlp.  The masks are never stored: every
// kernel (forward, recompute, backward) regenerates the keep/drop decision of an element from a counter hash of
// (seed, stream, element index) -- stream 0: edge hidden (pair, channel), 1: coors hidden (pair, unit), 2: node hidden
// (node, channel).  Statistically equivalent to the reference's Philox masks, not bit-equal (nothing could be).
// A kept unit is scaled by 1/(1-p) in the kernel's type, as nn.Dropout scales in the layer's dtype: the fp64 kernels
// use the double (float(1/(1-p)) differs from it by up to 5e-8 relative, e.g. at p = 0.1).
struct DropCfg {
  unsigned int thr;            // drop when hash < thr;  0 = dropout off
  float inv_keep;              // 1 / (1 - p) rounded to float: the fp32 kernels' scale
  unsigned long long seed;
  double inv_keep_d;           // 1 / (1 - p): the fp64 kernels' scale
};
__host__ __device__ inline DropCfg make_drop(double p, unsigned long long seed) {
  DropCfg d;
  d.thr = p > 0.0 ? (unsigned int)(p * 4294967296.0 > 4294967295.0 ? 4294967295.0 : p * 4294967296.0) : 0u;
  d.inv_keep_d = p > 0.0 && p < 1.0 ? 1.0 / (1.0 - p) : 1.0;
  d.inv_keep = (float)d.inv_keep_d;
  d.seed = seed;
  return d;
}
template <typename T> __device__ __forceinline__ T drop_scale(const DropCfg& d);
template <> __device__ __forceinline__ float drop_scale<float>(const DropCfg& d) { return d.inv_keep; }
template <> __device__ __forceinline__ double drop_scale<double>(const DropCfg& d) { return d.inv_keep_d; }
// multiplier of the pre-activation in type T: 0 (dropped) or 1/(1-p) (kept)
template <typename T>
__device__ __forceinline__ T drop_mul(const DropCfg& d, unsigned int stream, unsigned long long idx) {
  unsigned long long z = idx * 0x9E3779B97F4A7C15ull + d.seed + (unsigned long long)stream * 0xD1B54A32D192ED03ull;
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27; z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (unsigned int)(z >> 32) < d.thr ? T(0) : drop_scale<T>(d);
}

// ------------------------------------------------------------------ scalar math
template <typename T> __device__ __forceinline__ T silu_acc(T x);
template <> __device__ __forceinline__ float silu_acc<float>(float x) {
  // x * sigmoid(x): ex2.approx-based __expf (2 ulp) and rcp.approx-based __fdividef (2 ulp); for x < -88 the
  // denominator overflows to +inf and the quotient is -0, which is the correct limit.
  return __fdividef(x, 1.0f + __expf(-x));
}
template <> __device__ __forceinline__ double silu_acc<double>(double x) {
  return x / (1.0 + exp(-x));
}
// nn.GELU() (exact): 0.5 x (1 + erf(x / sqrt 2))   (GlobalLinearAttention's feed-forward, egnn_pytorch.py:127)
template <typename T> __device__ __forceinline__ T gelu_acc(T x);
template <> __device__ __forceinline__ float gelu_acc<float>(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
template <> __device__ __forceinline__ double gelu_acc<double>(double x) { return 0.5 * x * (1.0 + erf(x * 0.70710678118654752440)); }
template <typename T> __device__ __forceinline__ T sigmoid_acc(T x);
template <> __device__ __forceinline__ float sigmoid_acc<float>(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
template <> __device__ __forceinline__ double sigmoid_acc<double>(double x) { return 1.0 / (1.0 + exp(-x)); }

template <typename T> __device__ __forceinline__ T fma_t(T a, T b, T c);
template <> __device__ __forceinline__ float fma_t<float>(float a, float b, float c) { return fmaf(a, b, c); }
template <> __device__ __forceinline__ double fma_t<double>(double a, double b, double c) { return fma(a, b, c); }

// a*a + acc WITHOUT fma contraction: the reference forms (rel ** 2).sum(-1) (egnn_pytorch.py:233) with separate
// multiplies and adds, and neighbour ranking is sensitive to the last bit near the k-th boundary.
template <typename T> __device__ __forceinline__ T sq_acc(T a, T acc);
template <> __device__ __forceinline__ float sq_acc<float>(float a, float acc) { return __fadd_rn(acc, __fmul_rn(a, a)); }
template <> __device__ __forceinline__ double sq_acc<double>(double a, double acc) { return __dadd_rn(acc, __dmul_rn(a, a)); }

// ------------------------------------------------------------------ periodic boundaries (minimum image)
// Axis c of graph b's box as the kernels use it: the length L and 1/L, both 0 on an axis that is not periodic (L = 0
// or +inf) and beyond C, so that min_image leaves such an axis unchanged.  Read once per row or CTA, never per pair.
template <typename T>
__device__ __forceinline__ void box_axis(const T* box, int b, int C, int c, T& L, T& inv) {
  const T l = c < C ? box[(size_t)b * C + c] : T(0);
  const bool periodic = l > T(0) && l < T(INFINITY);
  L = periodic ? l : T(0);
  inv = periodic ? T(1) / l : T(0);
}
// rel - L rint(rel / L): the minimum-image difference (rounding half to even, as rintf / rint / np.rint)
template <typename T> __device__ __forceinline__ T min_image(T r, T L, T inv);
template <> __device__ __forceinline__ float min_image<float>(float r, float L, float inv) { return fmaf(-L, rintf(r * inv), r); }
template <> __device__ __forceinline__ double min_image<double>(double r, double L, double inv) { return fma(-L, rint(r * inv), r); }
// min_image with the same operations, also returning the image count n = rint(rel / L) it subtracts (0 on an aperiodic
// axis, where inv = 0), which the box gradient needs: rel = (x_i - x_j) - n L.
template <typename T> __device__ __forceinline__ T min_image_n(T r, T L, T inv, T& n) {
  n = rint(r * inv);
  return fma_t<T>(-L, n, r);
}

// ------------------------------------------------------------------ periodic boundaries (triclinic cells)
// The PBC template parameter of every kernel that forms x_i - x_j: no wrap, an orthorhombic box ([B,C] lengths), or a
// lower-triangular cell ([B,C,C], row k = lattice vector a_k, C in {2, 3}; DESIGN.md section 4).
constexpr int PBC_NONE = 0, PBC_BOX = 1, PBC_CELL = 2;
// A cell as the kernels stage it, once per CTA, row or ring slot: the diagonal L[3] and 1/L[3] exactly as box_axis
// forms them (0 on an aperiodic axis and beyond C), then the off-diagonals a_1x, a_2x, a_2y (0 beyond C).
constexpr int CELL_STAGED = 9;
template <typename T>
__device__ __forceinline__ T cell_staged(const T* cell, int b, int C, int t) {
  const T* m = cell + (size_t)b * C * C;
  if (t < 6) {
    const int c = t % 3;
    const T l = c < C ? m[c * C + c] : T(0);
    const bool periodic = l > T(0) && l < T(INFINITY);
    return !periodic ? T(0) : (t < 3 ? l : T(1) / l);
  }
  const int r = t == 6 ? 1 : 2, c = t == 8 ? 1 : 0;
  return r < C ? m[r * C + c] : T(0);
}
// The sequential wrap under a staged cell pc, from the last axis to the first: n = rint(r_c / L_c), then
// r_d -= cell[c][d] n for every d <= c.  Afterwards |r_c| <= L_c / 2 on every periodic axis.  With a diagonal cell
// the off-diagonal steps subtract exact zeros, so the result is min_image's bit for bit.  cell_wrap_n also returns the
// image counts n[c] (0 on an aperiodic axis): the wrapped vector is (x_i - x_j) - sum_c n[c] a_c, which the cell
// gradient needs.
template <typename T>
__device__ __forceinline__ void cell_wrap_n(T& r0, T& r1, T& r2, T (&n)[3], const T* pc) {
  n[2] = rint(r2 * pc[5]);
  r0 = fma_t<T>(-pc[7], n[2], r0); r1 = fma_t<T>(-pc[8], n[2], r1); r2 = fma_t<T>(-pc[2], n[2], r2);
  n[1] = rint(r1 * pc[4]);
  r0 = fma_t<T>(-pc[6], n[1], r0); r1 = fma_t<T>(-pc[1], n[1], r1);
  n[0] = rint(r0 * pc[3]);
  r0 = fma_t<T>(-pc[0], n[0], r0);
}
template <typename T>
__device__ __forceinline__ void cell_wrap(T& r0, T& r1, T& r2, const T* pc) {
  T n[3];
  cell_wrap_n<T>(r0, r1, r2, n, pc);
}

// 4 consecutive elements, 4-element aligned.
template <typename T> struct Vec4;
template <> struct Vec4<float> {
  float v[4];
  __device__ __forceinline__ void load(const float* p) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  __device__ __forceinline__ void load_g(const float* p) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
};
template <> struct Vec4<double> {
  double v[4];
  __device__ __forceinline__ void load(const double* p) {
    double2 a = *reinterpret_cast<const double2*>(p);
    double2 b = *reinterpret_cast<const double2*>(p + 2);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
  __device__ __forceinline__ void load_g(const double* p) {
    double2 a = __ldg(reinterpret_cast<const double2*>(p));
    double2 b = __ldg(reinterpret_cast<const double2*>(p + 2));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};

template <typename T> __device__ __forceinline__ T shfl_xor_t(T v, int m);
template <> __device__ __forceinline__ float shfl_xor_t<float>(float v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
template <> __device__ __forceinline__ double shfl_xor_t<double>(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
template <typename T> __device__ __forceinline__ T shfl_idx_t(T v, int l);
template <> __device__ __forceinline__ float shfl_idx_t<float>(float v, int l) { return __shfl_sync(0xffffffffu, v, l); }
template <> __device__ __forceinline__ double shfl_idx_t<double>(double v, int l) { return __shfl_sync(0xffffffffu, v, l); }

// ------------------------------------------------------------------ packed parameter layout (SIMT path)
// All offsets in elements of T; every block is 4-element aligned.
struct SimtPackLayout {
  size_t w2t;     // [Hp][MP]     W2 transposed, zero padded (MP = 16 or 32)
  size_t wq;      // [Q][Hp]      per-pair scalar columns of W1: distance features then edges
  size_t tab;     // [num_labels][Hp]  label_emb @ W1[:, label cols]^T
  size_t w3;      // [4m][MP]     coors_mlp.0.weight, padded
  size_t b3;      // [4m]
  size_t w4;      // [4m]
  size_t misc;    // b2[MP] | gate_w[MP] | gate_b | b4 | coors_scale | pad
  size_t total;
  int MP;
};

inline SimtPackLayout simt_pack_layout(const Dims& s) {
  SimtPackLayout L;
  L.MP = s.m <= 16 ? 16 : 32;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += round_up(n, 4); return r; };
  L.w2t = take((size_t)s.Hp * L.MP);
  L.wq = take((size_t)s.Q * s.Hp);
  L.tab = take((size_t)(s.label_dim > 0 ? s.num_labels : 0) * s.Hp);
  L.w3 = take((size_t)4 * s.m * L.MP);
  L.b3 = take((size_t)4 * s.m);
  L.w4 = take((size_t)4 * s.m);
  L.misc = take((size_t)2 * L.MP + 4);
  L.total = o;
  return L;
}

}  // namespace egnn

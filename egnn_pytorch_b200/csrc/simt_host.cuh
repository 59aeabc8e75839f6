// Host-side helpers shared by the forward (egnn_api.cu) and backward (egnn_backward.cu) orchestration:
// descriptor validation, the forward workspace layout and the GEMM launcher.
#pragma once
#include "common.cuh"
#include "simt_kernels.cuh"
#include "profile.h"
#include <algorithm>

namespace egnn {

// ------------------------------------------------------------------ validation
static int validate_desc(const EgnnLayerDesc* d) {
  if (!d) return EGNN_ERR_NULL;
  if (d->abi_version != EGNN_ABI_VERSION) return EGNN_ERR_ABI;
  if (d->dtype != EGNN_DTYPE_F32 && d->dtype != EGNN_DTYPE_F64 && d->dtype != EGNN_DTYPE_BF16)
    return EGNN_ERR_UNSUPPORTED;
  if (d->B <= 0 || d->N <= 0 || d->dim <= 0 || d->C <= 0 || d->edge_dim < 0 || d->label_dim < 0 ||
      d->fourier < 0 || d->m_dim <= 0 || d->k < 0)
    return EGNN_ERR_SHAPE;
  if (d->B > 65535) return EGNN_ERR_SHAPE;
  if (d->C > PAIR_CMAX) return EGNN_ERR_UNSUPPORTED;
  if (d->m_dim > 32) return EGNN_ERR_UNSUPPORTED;
  if (d->fourier > 30) return EGNN_ERR_UNSUPPORTED;
  if (d->k > d->N) return EGNN_ERR_SHAPE;                 // torch.topk raises too (:258)
  if (d->label_dim > 0 && (d->num_labels <= 0 || d->num_labels > 255)) return EGNN_ERR_SHAPE;
  if (!(d->flags & (EGNN_FLAG_UPDATE_FEATS | EGNN_FLAG_UPDATE_COORS))) return EGNN_ERR_SHAPE;   // :171
  if (d->reserved != 0) return EGNN_ERR_SHAPE;
  if (!(d->dropout_p >= 0.0 && d->dropout_p < 1.0)) return EGNN_ERR_SHAPE;
  if (d->dropout_p > 0.0 && d->dtype == EGNN_DTYPE_BF16) return EGNN_ERR_UNSUPPORTED;     // training runs the fp32 / fp64 kernels
  if (d->row_begin < 0 || d->row_end < 0 || d->row_end > d->N || d->row_begin > d->row_end) return EGNN_ERR_SHAPE;
  // per-slot edges follow the slots of caller-supplied lists; the library's own top-k has no order they could follow
  if ((d->flags & EGNN_FLAG_EDGES_PER_SLOT) && (d->k == 0 || d->edge_dim == 0)) return EGNN_ERR_SHAPE;
  return EGNN_OK;
}

static inline size_t elem_size(int dtype) { return dtype == EGNN_DTYPE_F64 ? 8 : (dtype == EGNN_DTYPE_F32 ? 4 : 2); }

// ------------------------------------------------------------------ SIMT workspace
struct SimtWs {
  size_t P, node_in, h1, nbr_idx, nbr_ok, hpart, cell, cell_bytes, total;
  int hsplit;
};
// Tiny dense graphs (the README example, BASELINE config 1): too few (row, neighbour) tiles to fill the GPU, so the
// hidden axis is split over CTAs and the partial sums take one trip through the workspace.
// cell_bytes: the cell-grid select's scratch (cell_select_layer_ws_bytes), placed last so that every other offset is
// the same with and without it (the backward reads the forward's regions at these offsets).
static int simt_hsplit(const Dims& s) {
  if (s.k != 0 || (long long)s.B * s.N * s.N > 4096 || s.Hp < 512 || s.row0 != 0 || s.row1 != s.N) return 1;
  return std::min(32, ceil_div(s.Hp, PAIR_CH));
}
static SimtWs simt_ws_layout(const Dims& s, size_t es, uint32_t flags, size_t cell_bytes = 0) {
  SimtWs w;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += round_up(bytes, 256); return r; };
  w.P = take((size_t)s.M * 2 * s.Hp * es);
  const bool uf = flags & EGNN_FLAG_UPDATE_FEATS;
  w.node_in = take(uf ? (size_t)s.M * (s.dim + s.m) * es : 0);
  w.h1 = take(uf ? (size_t)s.M * 2 * s.dim * es : 0);
  w.nbr_idx = take((size_t)s.M * s.k * sizeof(int32_t));
  w.nbr_ok = take((size_t)s.M * s.k);
  w.hsplit = simt_hsplit(s);
  w.hpart = take(w.hsplit > 1 ? (size_t)w.hsplit * s.B * s.N * s.N * 32 * es : 0);
  w.cell = take(cell_bytes);
  w.cell_bytes = cell_bytes;
  w.total = o;
  return w;
}

// Shared memory budget of the SIMT kernels.  A configuration over it is unsupported; the dense edge step then falls
// back from two rows per thread to one.
constexpr size_t SIMT_SMEM_MAX = 220 * 1024;

// Opt in, launch one SIMT kernel with `smem` bytes of dynamic shared memory, and check the enqueue.
template <typename Arg>
static int launch_simt(void (*kernel)(Arg), dim3 grid, int threads, size_t smem, cudaStream_t st, const Arg& arg) {
  if (smem > SIMT_SMEM_MAX) return EGNN_ERR_UNSUPPORTED;
  EGNN_TRY(ensure_dynamic_smem(kernel, smem));
  kernel<<<grid, threads, smem, st>>>(arg);
  EGNN_LAUNCH_CHECK();
  return EGNN_OK;
}

// The edge step over neighbour lists.  PBC: the periodic instantiations (a.box set).
template <typename T, int MP, int PBC = PBC_NONE>
static int launch_pair(const PairArgs<T>& a, cudaStream_t st) {
  dim3 grid(ceil_div(a.s.row1 - a.s.row0, PAIR_THREADS / a.TS), a.s.B);
  void (*kernel)(PairArgs<T>) = row_block(a.s, a.flags) ? pair_kernel<T, MP, true, PBC> : pair_kernel<T, MP, false, PBC>;
  return launch_simt(kernel, grid, PAIR_THREADS, pair_smem_bytes<T>(a.s, a.L), st, a);
}

// The dense edge step at PP rows per thread; a.hsplit > 1 runs it as two phases over a split hidden axis.
template <typename T, int MP, int PP, int PBC>
static int launch_pair_tiled(const PairArgs<T>& a, cudaStream_t st) {
  const size_t smem = pair_tiled_smem_bytes<T>(a.s, a.L, PP);
  dim3 grid(ceil_div(a.s.row1 - a.s.row0, 4 * PP), a.s.B);
  if (a.hsplit > 1) {                                 // (all rows only: simt_hsplit)
    PairArgs<T> a1 = a, a2 = a;
    a1.phase = 1; a2.phase = 2;
    a1.pre2_out = nullptr;                            // partial sums; phase 2 holds the full ones
    EGNN_TRY(launch_simt(pair_dense_tiled_kernel<T, MP, PP, false, PBC>, dim3(grid.x, grid.y, a.hsplit), PAIR_THREADS, smem, st, a1));
    return launch_simt(pair_dense_tiled_kernel<T, MP, PP, false, PBC>, grid, PAIR_THREADS, smem, st, a2);
  }
  void (*kernel)(PairArgs<T>) = row_block(a.s, a.flags) ? pair_dense_tiled_kernel<T, MP, PP, true, PBC>
                                                        : pair_dense_tiled_kernel<T, MP, PP, false, PBC>;
  return launch_simt(kernel, grid, PAIR_THREADS, smem, st, a);
}

// The dense edge step at two rows per thread where its shared memory fits, else at one (fp64 with m_dim > 16:
// one always).
template <typename T, int MP, int PBC = PBC_NONE>
static int launch_pair_dense(const PairArgs<T>& a, cudaStream_t st) {
  constexpr int PP = (MP == 32 && sizeof(T) == 8) ? 1 : 2;
  const int rc = launch_pair_tiled<T, MP, PP, PBC>(a, st);
  if (PP == 1 || rc != EGNN_ERR_UNSUPPORTED) return rc;
  return launch_pair_tiled<T, MP, 1, PBC>(a, st);
}

template <typename T, int ACT, bool RES>
static int launch_gemm(const T* A, int lda, const T* W, int ldw, const T* bias, const T* R, int ldr, T* C,
                       int ldo, int Mr, int Nv, int Nout, int K, RowMap map, cudaStream_t st, DropCfg drop = make_drop(0.0, 0ull)) {
  constexpr int V = 16 / (int)sizeof(T);
  const size_t skinny_smem = (size_t)16 * ((K + V - 1) / V * V) * sizeof(T);
  if (Mr <= 16 && skinny_smem <= 96 * 1024) {
    // columns per warp: as many as still give about one CTA per SM (the kernel is bound by weight streaming)
    int sms = 0;
    EGNN_TRY(sm_count(&sms));
    const int cols = Nout >= sms * SKINNY_WARPS * 4 ? 4 : (Nout >= sms * SKINNY_WARPS * 2 ? 2 : 1);
    const int grid = ceil_div(Nout, SKINNY_WARPS * cols);
    if (cols == 4) {
      EGNN_TRY(ensure_dynamic_smem(gemm_skinny_kernel<T, ACT, RES, 4>, skinny_smem));
      gemm_skinny_kernel<T, ACT, RES, 4><<<grid, SKINNY_WARPS * 32, skinny_smem, st>>>(A, lda, W, ldw, bias, R, ldr, C, ldo, Mr, Nv, Nout, K, map, drop);
    } else if (cols == 2) {
      EGNN_TRY(ensure_dynamic_smem(gemm_skinny_kernel<T, ACT, RES, 2>, skinny_smem));
      gemm_skinny_kernel<T, ACT, RES, 2><<<grid, SKINNY_WARPS * 32, skinny_smem, st>>>(A, lda, W, ldw, bias, R, ldr, C, ldo, Mr, Nv, Nout, K, map, drop);
    } else {
      EGNN_TRY(ensure_dynamic_smem(gemm_skinny_kernel<T, ACT, RES, 1>, skinny_smem));
      gemm_skinny_kernel<T, ACT, RES, 1><<<grid, SKINNY_WARPS * 32, skinny_smem, st>>>(A, lda, W, ldw, bias, R, ldr, C, ldo, Mr, Nv, Nout, K, map, drop);
    }
    EGNN_LAUNCH_CHECK();
    count_launch();
    return EGNN_OK;
  }
  dim3 grid(ceil_div(Nout, 64), ceil_div(Mr, 64));
  gemm_nt_kernel<T, ACT, RES><<<grid, 256, 0, st>>>(A, lda, W, ldw, bias, R, ldr, C, ldo, Mr, Nv, Nout, K, map, drop);
  EGNN_LAUNCH_CHECK();
  count_launch();
  return EGNN_OK;
}

static int check_ptrs(const EgnnLayerDesc& d, const EgnnLayerWeights* w, const EgnnLayerIO* io) {
  if (!w || !w->edge_w1 || !w->edge_b1 || !w->edge_w2 || !w->edge_b2) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_SOFT_EDGES) && (!w->gate_w || !w->gate_b)) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_NORM_FEATS) && (d.flags & EGNN_FLAG_UPDATE_FEATS) && (!w->norm_g || !w->norm_b)) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_NORM_COORS) && !w->coors_scale) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_UPDATE_FEATS) && (!w->node_w1 || !w->node_b1 || !w->node_w2 || !w->node_b2)) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_UPDATE_COORS) && (!w->coors_w1 || !w->coors_b1 || !w->coors_w2 || !w->coors_b2)) return EGNN_ERR_NULL;
  if (d.label_dim > 0 && !w->label_emb) return EGNN_ERR_NULL;
  if (io) {
    if (!io->feats || !io->coors || !io->feats_out || !io->coors_out) return EGNN_ERR_NULL;
    if (d.edge_dim > 0 && !io->edges) return EGNN_ERR_NULL;
    if (d.label_dim > 0 && !io->edge_labels) return EGNN_ERR_NULL;
    if ((d.flags & EGNN_FLAG_EDGES_PER_SLOT) && !io->nbr_idx) return EGNN_ERR_SHAPE;
    const uintptr_t all = (uintptr_t)io->feats | (uintptr_t)io->feats_out | (uintptr_t)io->edges;
    if (all & 0xF) return EGNN_ERR_ALIGN;
  }
  return EGNN_OK;
}

}  // namespace egnn

#pragma once
// Per-layer backward orchestration (templated on the element type; instantiated once per type in
// egnn_backward.cu (fp32) and egnn_backward_f64.cu (fp64) so the two compile concurrently):
//   node update reversed -> bwd1 / bwd2 / bwd3 (simt_backward.cuh) -> per-node tables reversed -> unpack.
#include "common.cuh"
#include "simt_kernels.cuh"
#include "simt_backward.cuh"
#include "simt_host.cuh"

namespace egnn {

struct BwdWs {
  size_t gP, gpk, rec, pre2, h1pre, ga, g_node_in, gyx, total;
};

inline BwdWs bwd_ws_layout(const Dims& s, const SimtPackLayout& L, size_t es, uint32_t flags) {
  BwdWs w;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += round_up(bytes, 256); return r; };
  const size_t J = s.k > 0 ? s.k : s.N;
  const size_t Mp = (size_t)s.B * pair_rows(s, flags);           // rows of the per-pair buffers: all of them, or a row block's
  const bool uf = flags & EGNN_FLAG_UPDATE_FEATS;
  w.gP = take((size_t)s.M * 2 * s.Hp * es);
  w.gpk = take(L.total * es);
  w.rec = take(Mp * J * rec_layout(s, L.MP).R * es);
  w.pre2 = take(Mp * J * L.MP * es);
  w.h1pre = take(uf ? (size_t)s.M * 2 * s.dim * es : 0);
  w.ga = take(uf ? (size_t)s.M * 2 * s.dim * es : 0);
  w.g_node_in = take(uf ? (size_t)s.M * (s.dim + s.m) * es : 0);
  w.gyx = take((uf && (flags & EGNN_FLAG_NORM_FEATS)) ? (size_t)s.M * s.dim * es : 0);
  w.total = o;
  return w;
}

// Shared memory of bwd1 and bwd2, sized by the functions their launches use (launch_pair_bwd).
template <typename T>
inline bool backward_smem_fits(const Dims& s, uint32_t flags) {
  const SimtPackLayout L = simt_pack_layout(s);
  const int R = rec_layout(s, L.MP).R;
  const size_t bwd1 = bwd1_smem_bytes<T>(s, L, (flags & EGNN_FLAG_SOFT_EDGES) != 0);
  const size_t bwd2 = s.k > 0 ? bwd2_knn_smem_bytes<T>(s, R) : bwd2_dense_smem_bytes<T>(s, R);
  return bwd1 <= SIMT_SMEM_MAX && bwd2 <= SIMT_SMEM_MAX;
}

// Everything the backward kernels cannot run.  The training forward calls this first (through
// egnn_layer_backward_workspace_bytes), so such a configuration fails before the forward instead of in the backward.
inline int backward_supported(const EgnnLayerDesc& d) {
  if (d.dtype != EGNN_DTYPE_F32 && d.dtype != EGNN_DTYPE_F64) return EGNN_ERR_UNSUPPORTED;
  // a row block trains only as an explicit request for its partial gradients
  const bool all_rows = d.row_begin == 0 && (d.row_end == 0 || d.row_end == d.N);
  if (!all_rows && !(d.flags & EGNN_FLAG_ROW_PARTIAL_GRADS)) return EGNN_ERR_UNSUPPORTED;
  if (d.label_dim > 0 && d.num_labels > BW2_MAXLAB) return EGNN_ERR_UNSUPPORTED;
  const Dims s = make_dims(d);
  const bool fits = d.dtype == EGNN_DTYPE_F64 ? backward_smem_fits<double>(s, d.flags) : backward_smem_fits<float>(s, d.flags);
  if (!fits) return EGNN_ERR_UNSUPPORTED;
  return EGNN_OK;
}

// The node rows of a row block, r -> b * N + row0 + r % R; the identity for the full range.
static inline bool is_identity(const RowMap& m) { return m.Rr == m.N && m.row0 == 0; }

// C[r,c] += sum_k A(r,k) B(k,c); K is split so that small outputs with a long reduction still fill the GPU.  `axis`
// (ACC_ROWS / ACC_K) names the index that runs over node rows when `map` selects a row block.
template <typename T>
static int launch_gemm_acc(const T* A, long ars, long aks, const T* B, long bks, long bcs, T* C, long ldc, int Mr,
                           int Nc, int K, cudaStream_t st, RowMap map = RowMap{1, 1, 0}, int axis = ACC_PLAIN) {
  if (Mr <= 0 || Nc <= 0 || K <= 0) return EGNN_OK;
  const int tiles = ceil_div(Mr, 64) * ceil_div(Nc, 64);
  int sms = 0;
  EGNN_TRY(sm_count(&sms));
  int splits = std::max(1, std::min(ceil_div(2 * sms, tiles), ceil_div(K, 64)));     // about two CTAs per SM
  splits = std::min(splits, 65535);
  const int kper = round_up_i(ceil_div(K, splits), 16);
  splits = ceil_div(K, kper);
  dim3 grid(ceil_div(Nc, 64), ceil_div(Mr, 64), splits);
  if (is_identity(map)) axis = ACC_PLAIN;
  if (axis == ACC_ROWS) gemm_acc_kernel<T, ACC_ROWS><<<grid, 256, 0, st>>>(A, ars, aks, B, bks, bcs, C, ldc, Mr, Nc, K, kper, map);
  else if (axis == ACC_K) gemm_acc_kernel<T, ACC_K><<<grid, 256, 0, st>>>(A, ars, aks, B, bks, bcs, C, ldc, Mr, Nc, K, kper, map);
  else gemm_acc_kernel<T, ACC_PLAIN><<<grid, 256, 0, st>>>(A, ars, aks, B, bks, bcs, C, ldc, Mr, Nc, K, kper, map);
  EGNN_LAUNCH_CHECK();
  return EGNN_OK;
}

template <typename T>
static int launch_colsum(const T* X, long ld, int rows, int cols, T* out, cudaStream_t st, RowMap map = RowMap{1, 1, 0}) {
  if (rows <= 0 || cols <= 0) return EGNN_OK;
  dim3 grid(ceil_div(cols, 32), std::max(1, std::min(64, ceil_div(rows, 64))));
  if (is_identity(map)) colsum_acc_kernel<T, false><<<grid, dim3(32, 8), 0, st>>>(X, ld, rows, cols, out, map);
  else colsum_acc_kernel<T, true><<<grid, dim3(32, 8), 0, st>>>(X, ld, rows, cols, out, map);
  EGNN_LAUNCH_CHECK();
  return EGNN_OK;
}

// W2 silu(pre1) of every pair into pre2 when the forward did not keep it, by the forward's own edge kernels (with
// the forward's dropout masks): for dense graphs the register-tiled kernel's split-H phase 1 over one split, which
// stores exactly that; for neighbour lists pair_kernel with no node or coordinate update.
template <typename T, int MP, int PBC>
static int recompute_pre2(const BwdArgs<T>& a, T* pre2, cudaStream_t st) {
  PairArgs<T> f;
  f.s = a.s; f.L = a.L; f.flags = a.flags; f.has_mask = a.has_mask; f.TS = a.TS; f.clamp = a.clamp;
  f.P = a.P; f.ldP = a.ldP; f.coors = a.coors; f.edges = a.edges; f.labels = a.labels; f.mask = a.mask;
  f.nbr_idx = a.nbr_idx; f.nbr_ok = a.nbr_ok; f.packed = a.packed;
  f.m_out = nullptr; f.ld_m = 0; f.coors_out = nullptr;
  f.hpart = nullptr; f.hsplit = 1; f.phase = 0;
  f.pre2_out = nullptr;
  f.drop = a.drop;
  f.box = a.box;
  if (a.s.k > 0) {
    f.flags &= ~(uint32_t)(EGNN_FLAG_UPDATE_FEATS | EGNN_FLAG_UPDATE_COORS);
    f.pre2_out = pre2;
    return launch_pair<T, MP, PBC>(f, st);
  }
  f.hpart = pre2; f.phase = 1;
  return launch_pair_dense<T, MP, PBC>(f, st);
}

// BLK: a row block (its own instantiations, so that the whole-graph kernels keep their plain row arithmetic).
// PBC: periodic geometry in bwd1 / bwd3 (bwd2 reads the pair records only).
template <typename T, int MP, bool KNN, bool BLK, int PBC>
static int launch_pair_bwd(const BwdArgs<T>& a, cudaStream_t st) {
  const Dims& s = a.s;
  const int rows = s.row1 - s.row0;                 // the i-rows of the call (all N unless a row block); the last CTA
                                                    // of each grid masks the rows past row1
  const dim3 g1(ceil_div(rows, PAIR_THREADS / a.TS), s.B);
  EGNN_TRY(launch_simt(pair_bwd1_kernel<T, MP, KNN, BLK, PBC>, g1, PAIR_THREADS,
                       bwd1_smem_bytes<T>(s, a.L, (a.flags & EGNN_FLAG_SOFT_EDGES) != 0), st, a));
  // bwd2: distance channel only (QR = 1), up to 8 channels in registers (lists only, QR = 8) or any (QR = 0); the
  // dropout masks in their own instantiations
  const bool simple = s.Q == 1 && s.label_dim == 0, drop = a.drop.thr != 0;
  void (*bwd2)(BwdArgs<T>);
  size_t smem2;
  dim3 g2;
  if constexpr (KNN) {
    smem2 = bwd2_knn_smem_bytes<T>(s, a.rl.R);
    g2 = dim3(ceil_div(rows, a.TI2), ceil_div(s.Hp, BW2_TH), s.B);
    if (simple) bwd2 = drop ? pair_bwd2_knn_kernel<T, MP, 1, true, BLK> : pair_bwd2_knn_kernel<T, MP, 1, false, BLK>;
    else if (s.Q <= 8) bwd2 = drop ? pair_bwd2_knn_kernel<T, MP, 8, true, BLK> : pair_bwd2_knn_kernel<T, MP, 8, false, BLK>;
    else bwd2 = drop ? pair_bwd2_knn_kernel<T, MP, 0, true, BLK> : pair_bwd2_knn_kernel<T, MP, 0, false, BLK>;
  } else {
    smem2 = bwd2_dense_smem_bytes<T>(s, a.rl.R);
    g2 = dim3(ceil_div(rows, BW2_ROWS), ceil_div(s.Hp, BW2_TH), s.B);
    if (simple) bwd2 = drop ? pair_bwd2_dense_kernel<T, MP, 1, true, BLK> : pair_bwd2_dense_kernel<T, MP, 1, false, BLK>;
    else bwd2 = drop ? pair_bwd2_dense_kernel<T, MP, 0, true, BLK> : pair_bwd2_dense_kernel<T, MP, 0, false, BLK>;
  }
  EGNN_TRY(launch_simt(bwd2, g2, BW2_TH, smem2, st, a));
  bool lat = false;
  if constexpr (PBC != PBC_NONE) {     // the lattice gradient: its own bwd3 instantiation, launched only when asked for
    lat = a.g_lat != nullptr;
    if (lat) pair_bwd3_kernel<T, KNN, BLK, PBC, true><<<g1, PAIR_THREADS, 0, st>>>(a);
  }
  if (!lat) pair_bwd3_kernel<T, KNN, BLK, PBC><<<g1, PAIR_THREADS, 0, st>>>(a);
  EGNN_LAUNCH_CHECK();
  return EGNN_OK;
}

// The edge step reversed for one choice of (row block, neighbour lists, periodic box or cell).
template <typename T, int PBC>
static int launch_edge_bwd(const BwdArgs<T>& a, T* pre2, bool saved, bool part, cudaStream_t st) {
  const int MP = a.L.MP;
  if (!saved) EGNN_TRY((MP == 16 ? recompute_pre2<T, 16, PBC>(a, pre2, st) : recompute_pre2<T, 32, PBC>(a, pre2, st)));
  if (part) {
    if (a.s.k > 0) return MP == 16 ? launch_pair_bwd<T, 16, true, true, PBC>(a, st) : launch_pair_bwd<T, 32, true, true, PBC>(a, st);
    return MP == 16 ? launch_pair_bwd<T, 16, false, true, PBC>(a, st) : launch_pair_bwd<T, 32, false, true, PBC>(a, st);
  }
  if (a.s.k > 0) return MP == 16 ? launch_pair_bwd<T, 16, true, false, PBC>(a, st) : launch_pair_bwd<T, 32, true, false, PBC>(a, st);
  return MP == 16 ? launch_pair_bwd<T, 16, false, false, PBC>(a, st) : launch_pair_bwd<T, 32, false, false, PBC>(a, st);
}

// g_lat: null, or the fp64 lattice gradient ([B,C] for a box, [B,C,C] for a cell), overwritten.
template <typename T>
int simt_backward(const EgnnLayerDesc& d, const EgnnLayerWeights& w, const void* packed, const EgnnLayerIO& io,
                  const void* box, int pbc, const void* fwd_ws, const EgnnLayerGrads& gr, double* g_lat, void* ws,
                  size_t ws_bytes, cudaStream_t st) {
  const Dims s = make_dims(d);
  const SimtPackLayout L = simt_pack_layout(s);
  const SimtWs fl = simt_ws_layout(s, sizeof(T), d.flags);
  const BwdWs bl = bwd_ws_layout(s, L, sizeof(T), d.flags);
  if (ws_bytes < bl.total) return EGNN_ERR_WORKSPACE;
  const bool uf = d.flags & EGNN_FLAG_UPDATE_FEATS, uc = d.flags & EGNN_FLAG_UPDATE_COORS;
  const bool nf = d.flags & EGNN_FLAG_NORM_FEATS;
  const char* fbase = static_cast<const char*>(fwd_ws);
  char* base = static_cast<char*>(ws);
  const T* P = reinterpret_cast<const T*>(fbase + fl.P);
  const T* node_in = reinterpret_cast<const T*>(fbase + fl.node_in);
  const T* h1 = reinterpret_cast<const T*>(fbase + fl.h1);
  const int32_t* nbr_idx = reinterpret_cast<const int32_t*>(fbase + fl.nbr_idx);
  const uint8_t* nbr_ok = reinterpret_cast<const uint8_t*>(fbase + fl.nbr_ok);
  if (s.k > 0 && io.nbr_idx) { nbr_idx = io.nbr_idx; nbr_ok = nullptr; }
  T* gP = reinterpret_cast<T*>(base + bl.gP);
  T* gpk = reinterpret_cast<T*>(base + bl.gpk);
  T* rec = reinterpret_cast<T*>(base + bl.rec);
  T* h1pre = reinterpret_cast<T*>(base + bl.h1pre);
  T* ga = reinterpret_cast<T*>(base + bl.ga);
  T* g_node_in = reinterpret_cast<T*>(base + bl.g_node_in);
  T* gyx = reinterpret_cast<T*>(base + bl.gyx);
  const T* feats = static_cast<const T*>(io.feats);
  const T* W1 = static_cast<const T*>(w.edge_w1);
  const T* go = static_cast<const T*>(gr.g_feats_out);
  T* g_feats = static_cast<T*>(gr.g_feats);
  T* g_coors = static_cast<T*>(gr.g_coors);
  const int M = s.M, dim = s.dim, m = s.m, dn = s.dim + s.m, d2 = 2 * s.dim;
  const size_t J = s.k > 0 ? s.k : s.N;
  // The i-rows differentiated: all of them, or a row block under EGNN_FLAG_ROW_PARTIAL_GRADS (backward_supported).  The
  // forward wrote node_in, h1 and the pooled messages of these rows only, so every node-level step of the block runs
  // over its Mb rows through `blk` -- the other rows of the forward workspace are uninitialised (NaN * 0 is NaN).
  const int Rb = s.row1 - s.row0, Mb = s.B * Rb;
  const RowMap blk{Rb, s.N, s.row0};
  const bool part = !is_identity(blk);

  // ---- zero the accumulators and the parameter-gradient outputs
  auto zero = [&](void* p, size_t bytes) -> int {
    if (p && bytes) EGNN_CUDA_TRY(cudaMemsetAsync(p, 0, bytes, st));
    return EGNN_OK;
  };
  const size_t es = sizeof(T);
  EGNN_TRY(zero(gP, (size_t)M * 2 * s.Hp * es));
  EGNN_TRY(zero(gpk, L.total * es));
  EGNN_TRY(zero(rec, (size_t)s.B * pair_rows(s, d.flags) * J * rec_layout(s, L.MP).R * es));
  EGNN_TRY(zero(gr.w.edge_w1, (size_t)s.H * s.E * es));
  EGNN_TRY(zero(gr.w.edge_b1, (size_t)s.H * es));
  EGNN_TRY(zero(gr.w.edge_w2, (size_t)m * s.H * es));
  EGNN_TRY(zero(gr.w.edge_b2, (size_t)m * es));
  EGNN_TRY(zero(gr.w.gate_w, (size_t)m * es));
  EGNN_TRY(zero(gr.w.gate_b, es));
  EGNN_TRY(zero(gr.w.norm_g, (size_t)dim * es));
  EGNN_TRY(zero(gr.w.norm_b, (size_t)dim * es));
  EGNN_TRY(zero(gr.w.coors_scale, es));
  EGNN_TRY(zero(gr.w.node_w1, (size_t)d2 * dn * es));
  EGNN_TRY(zero(gr.w.node_b1, (size_t)d2 * es));
  EGNN_TRY(zero(gr.w.node_w2, (size_t)dim * d2 * es));
  EGNN_TRY(zero(gr.w.node_b2, (size_t)dim * es));
  EGNN_TRY(zero(gr.w.coors_w1, (size_t)4 * m * m * es));
  EGNN_TRY(zero(gr.w.coors_b1, (size_t)4 * m * es));
  EGNN_TRY(zero(gr.w.coors_w2, (size_t)4 * m * es));
  EGNN_TRY(zero(gr.w.coors_b2, es));
  EGNN_TRY(zero(gr.w.label_emb, (size_t)s.num_labels * s.label_dim * es));
  if (box) EGNN_TRY(zero(g_lat, (size_t)s.B * s.C * (pbc == PBC_CELL ? s.C : 1) * sizeof(double)));
  // neighbour lists: bwd3 adds dL/d edges into [B,N,N,e] with atomics, or stores them per slot ([B,N,k,e]) -- empty slots
  // are skipped, so they keep these zeros
  const size_t edge_rows = (d.flags & EGNN_FLAG_EDGES_PER_SLOT) ? (size_t)s.k : (size_t)s.N;
  if (gr.g_edges && s.k > 0) EGNN_TRY(zero(gr.g_edges, (size_t)M * edge_rows * s.edge_dim * es));
  // residual / identity paths: h' = ... + h (:337, :339), x' = x + ... (:315, :317) -- the same with update_feats /
  // update_coors off, where the output is the input
  if (!part) {
    EGNN_CUDA_TRY(cudaMemcpyAsync(g_feats, go, (size_t)M * dim * es, cudaMemcpyDeviceToDevice, st));
    EGNN_CUDA_TRY(cudaMemcpyAsync(g_coors, gr.g_coors_out, (size_t)M * s.C * es, cudaMemcpyDeviceToDevice, st));
  } else {
    // a row block: its own rows of the cotangents, 0 elsewhere; dense dL/d edges, which bwd3 stores for the block's
    // pairs only, is 0 in the other rows
    EGNN_TRY(zero(g_feats, (size_t)M * dim * es));
    EGNN_TRY(zero(g_coors, (size_t)M * s.C * es));
    auto copy_rows = [&](void* dst, const void* src, int width) -> int {
      const size_t pitch = (size_t)s.N * width * es, off = (size_t)s.row0 * width * es;
      if (Rb > 0)
        EGNN_CUDA_TRY(cudaMemcpy2DAsync(static_cast<char*>(dst) + off, pitch, static_cast<const char*>(src) + off, pitch,
                                        (size_t)Rb * width * es, s.B, cudaMemcpyDeviceToDevice, st));
      return EGNN_OK;
    };
    EGNN_TRY(copy_rows(g_feats, go, dim));
    EGNN_TRY(copy_rows(g_coors, gr.g_coors_out, s.C));
    if (gr.g_edges && s.k == 0) {
      const size_t row_bytes = (size_t)s.N * s.edge_dim * es, pitch = (size_t)s.N * row_bytes;
      char* ge = static_cast<char*>(gr.g_edges);
      if (s.row0 > 0) EGNN_CUDA_TRY(cudaMemset2DAsync(ge, pitch, 0, (size_t)s.row0 * row_bytes, s.B, st));
      if (s.row1 < s.N)
        EGNN_CUDA_TRY(cudaMemset2DAsync(ge + (size_t)s.row1 * row_bytes, pitch, 0, (size_t)(s.N - s.row1) * row_bytes, s.B, st));
    }
  }
  if (Rb == 0) return EGNN_OK;                       // an empty block: every gradient is the zero written above

  // ---- node update reversed (egnn_pytorch.py:335-337)
  if (uf) {
    const T* Wn1 = static_cast<const T*>(w.node_w1);
    const T* Wn2 = static_cast<const T*>(w.node_w2);
    EGNN_TRY(zero(ga, (size_t)M * d2 * es));
    EGNN_TRY(zero(g_node_in, (size_t)M * dn * es));
    EGNN_TRY((launch_gemm<T, 0, false>(node_in, dn, Wn1, dn, static_cast<const T*>(w.node_b1), nullptr, 0, h1pre, d2, Mb,
                                       d2, d2, dn, blk, st)));
    // dWn2[n][k] = sum_r go[r][n] h1[r][k];  db2 = colsum(go);  ga = go Wn2
    EGNN_TRY(launch_gemm_acc<T>(go, 1, dim, h1, d2, 1, static_cast<T*>(gr.w.node_w2), d2, dim, d2, Mb, st, blk, ACC_K));
    EGNN_TRY(launch_colsum<T>(go, dim, Mb, dim, static_cast<T*>(gr.w.node_b2), st, blk));
    EGNN_TRY(launch_gemm_acc<T>(go, dim, 1, Wn2, d2, 1, ga, d2, Mb, d2, dim, st, blk, ACC_ROWS));
    const int dgrid = (int)std::min<size_t>(2048, ((size_t)Mb * d2 + 255) / 256);
    const DropCfg ndrop = make_drop(d.dropout_p, d.dropout_seed);
    if (part) dsilu_mul_kernel<T, true><<<dgrid, 256, 0, st>>>(ga, h1pre, (size_t)Mb * d2, d2, blk, ndrop);
    else dsilu_mul_kernel<T, false><<<dgrid, 256, 0, st>>>(ga, h1pre, (size_t)M * d2, d2, blk, ndrop);
    EGNN_LAUNCH_CHECK();
    // dWn1[k][c] = sum_r gh1[r][k] node_in[r][c];  db1 = colsum(gh1);  g_node_in = gh1 Wn1
    EGNN_TRY(launch_gemm_acc<T>(ga, 1, d2, node_in, dn, 1, static_cast<T*>(gr.w.node_w1), dn, d2, dn, Mb, st, blk, ACC_K));
    EGNN_TRY(launch_colsum<T>(ga, d2, Mb, d2, static_cast<T*>(gr.w.node_b1), st, blk));
    EGNN_TRY(launch_gemm_acc<T>(ga, d2, 1, Wn1, dn, 1, g_node_in, dn, Mb, dn, d2, st, blk, ACC_ROWS));
    const T* lng = static_cast<const T*>(w.norm_g);
    if (part) ln_bwd_kernel<T, true><<<ceil_div(Mb * 32, 256), 256, 0, st>>>(feats, lng, g_node_in, dn, g_feats, gyx, dim, Mb, nf ? 1 : 0, blk);
    else ln_bwd_kernel<T, false><<<ceil_div(M * 32, 256), 256, 0, st>>>(feats, lng, g_node_in, dn, g_feats, gyx, dim, M, nf ? 1 : 0, blk);
    EGNN_LAUNCH_CHECK();
    if (nf) {
      EGNN_TRY(launch_colsum<T>(gyx, dim, Mb, dim, static_cast<T*>(gr.w.norm_g), st, blk));
      EGNN_TRY(launch_colsum<T>(g_node_in, dn, Mb, dim, static_cast<T*>(gr.w.norm_b), st, blk));
    }
  }

  // ---- the edge step reversed
  BwdArgs<T> a;
  a.s = s; a.L = L; a.rl = rec_layout(s, L.MP); a.flags = d.flags; a.has_mask = io.mask != nullptr;
  a.clamp = (T)d.clamp;
  a.P = P; a.ldP = 2 * s.Hp;
  a.coors = static_cast<const T*>(io.coors);
  a.edges = static_cast<const T*>(io.edges);
  a.labels = s.label_dim > 0 ? io.edge_labels : nullptr;
  a.mask = io.mask;
  a.nbr_idx = nbr_idx; a.nbr_ok = nbr_ok;
  a.packed = static_cast<const T*>(packed);
  a.g_node_in = uf ? g_node_in : nullptr; a.ld_g = dn;
  a.g_coors_out = static_cast<const T*>(gr.g_coors_out);
  a.drop = make_drop(d.dropout_p, d.dropout_seed);
  const bool saved = io.pre2_out != nullptr;                 // the forward kept W2 silu(pre1) per pair
  T* pre2 = saved ? static_cast<T*>(io.pre2_out) : reinterpret_cast<T*>(base + bl.pre2);
  a.pre2 = pre2;
  a.rec = rec; a.gpk = gpk; a.gP = gP; a.g_coors = g_coors;
  a.g_edges = (s.edge_dim > 0) ? static_cast<T*>(gr.g_edges) : nullptr;
  if (s.k > 0) {
    int TS = 1;
    while (TS < s.k && TS < 32) TS <<= 1;
    a.TS = TS; a.TI2 = 16;
  } else {
    a.TS = 32; a.TI2 = 32;
  }
  a.box = static_cast<const T*>(box);
  a.g_lat = box ? g_lat : nullptr;
  if (box && pbc == PBC_CELL) EGNN_TRY((launch_edge_bwd<T, PBC_CELL>(a, pre2, saved, part, st)));
  else if (box) EGNN_TRY((launch_edge_bwd<T, PBC_BOX>(a, pre2, saved, part, st)));
  else EGNN_TRY((launch_edge_bwd<T, PBC_NONE>(a, pre2, saved, part, st)));

  // ---- per-node tables reversed: A = h W1[:, :dim]^T + b1, B = h W1[:, dim:2dim]^T.  dL/dA is 0 outside the row block,
  // so its terms run over the block's rows; dL/dB (every j) over all rows
  T* gW1 = static_cast<T*>(gr.w.edge_w1);
  const int ldP = 2 * s.Hp;
  EGNN_TRY(launch_gemm_acc<T>(gP, ldP, 1, W1, s.E, 1, g_feats, dim, Mb, dim, s.H, st, blk, ACC_ROWS));  // g_h += gA W1_i
  EGNN_TRY(launch_gemm_acc<T>(gP + s.Hp, ldP, 1, W1 + dim, s.E, 1, g_feats, dim, M, dim, s.H, st));    // g_h += gB W1_j
  EGNN_TRY(launch_gemm_acc<T>(gP, 1, ldP, feats, dim, 1, gW1, s.E, s.H, dim, Mb, st, blk, ACC_K));      // dW1_i = gA^T h
  EGNN_TRY(launch_gemm_acc<T>(gP + s.Hp, 1, ldP, feats, dim, 1, gW1 + dim, s.E, s.H, dim, M, st));      // dW1_j = gB^T h
  EGNN_TRY(launch_colsum<T>(gP, ldP, Mb, s.H, static_cast<T*>(gr.w.edge_b1), st, blk));                 // db1

  int sms = 0;
  EGNN_TRY(sm_count(&sms));
  unpack_grads_kernel<T><<<sms, 256, 0, st>>>(s, L, d.flags, gpk, W1, static_cast<const T*>(w.label_emb), gr.w);
  EGNN_LAUNCH_CHECK();
  (void)uc; (void)h1;
  return EGNN_OK;
}

}  // namespace egnn

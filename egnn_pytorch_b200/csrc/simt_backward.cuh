// Backward of the EGNN layer (SIMT fp32 / fp64), SURVEY.md section 8(f) rank 1.
//
// The reference trains through autograd over the materialised [B,N,J,2E] tensors (egnn_pytorch.py:224-341).
// Here the forward is differentiated by hand in the split form of simt_kernels.cuh.  W2 silu(pre1) per pair (pre2)
// comes from the forward (EgnnLayerIO.pre2_out) or is recomputed before bwd1 by a forward kernel that stores it:
// the register-tiled kernel for dense graphs, pair_kernel for neighbour lists.
//
//   bwd1  thread per (i, slot) pair: from pre2, recompute m_ij, differentiate the pair epilogue (coordinate MLP, CoorsNorm,
//         clamp, masks, gate, pooling) and leave per pair  g_pre2[m] = dL/d(W2 hid + b2), the scalar channels f_q,
//         coef = w_ij * scale and the CoorsNorm part of dL/d(dist)  in a [pairs][R] record; the small parameter
//         gradients (coors_mlp, edge_gate, b2, coors_norm.scale) are reduced per CTA.
//   bwd2  thread per hidden channel h, CTA = (block of i rows) x (128 channels): for every pair recompute
//         pre1[h], hid[h]; g_hid = W2[:,h] . g_pre2; g_pre1 = g_hid * silu'(pre1).  Row sums give dL/dA_i, column
//         sums dL/dB_j, and  dL/dW2, dL/dWq, dL/dTab  accumulate in registers / shared memory; dL/df_q per pair is
//         reduced over h and added to the record.
//   bwd3  thread per pair: dL/d(dist) -> dL/d(rel) -> coordinates (x_i +, x_j -), dL/d(edges).
//
// The per-node GEMMs around them (tables A/B, node MLP, LayerNorm) are differentiated in egnn_backward.cu.
// Nothing of size O(pairs * H) is stored; the record is O(pairs * (m + 2Q + 2)).
#pragma once

#include "common.cuh"
#include "simt_kernels.cuh"

namespace egnn {

template <typename T> __device__ __forceinline__ void atomic_add_t(T* p, T v) { atomicAdd(p, v); }

struct RecLayout {
  int gpre2, f, gf, coef, gdn, R;
};
inline RecLayout rec_layout(const Dims& s, int MP) {
  RecLayout r;
  r.gpre2 = 0;
  r.f = MP;
  r.gf = MP + s.Q;
  r.coef = MP + 2 * s.Q;
  r.gdn = r.coef + 1;
  r.R = round_up_i(r.gdn + 1, 4);
  return r;
}

template <typename T>
struct BwdArgs {
  Dims s;
  SimtPackLayout L;
  RecLayout rl;
  uint32_t flags;
  int has_mask;
  int TS;                     // bwd1 / bwd3: slots per row group
  int TI2;                    // bwd2: rows per CTA
  T clamp;
  const T* P; int ldP;        // forward tables [M][2*Hp]: A | B
  const T* coors;
  const T* edges;                 // [B,N,N,edge_dim], [B,N,k,edge_dim] under EGNN_FLAG_EDGES_PER_SLOT, | null
  const uint8_t* labels;
  const uint8_t* mask;
  const int32_t* nbr_idx;
  const uint8_t* nbr_ok;
  const T* packed;
  const T* g_node_in; int ld_g;   // [M][dim+m]; dL/dm_i = columns dim..dim+m  (null when !update_feats)
  const T* g_coors_out;           // [B,N,C]
  const T* pre2;                  // W2 silu(pre1) per pair, row-major [B,N,J][MP] (rows by pair_row): saved by the forward
                                  // (EgnnLayerIO.pre2_out) or recomputed into the backward workspace
  T* rec;                         // [pairs][R]
  T* gpk;                         // gradient accumulators in SimtPackLayout order (zeroed by the caller)
  T* gP;                          // [M][2*Hp]: dL/dA | dL/dB (zeroed by the caller)
  T* g_coors;                     // [B,N,C], pre-loaded with g_coors_out
  T* g_edges;                     // [B,N,N,edge_dim], [B,N,k,edge_dim] under EGNN_FLAG_EDGES_PER_SLOT, | null
  DropCfg drop;                   // the forward's dropout configuration (masks are regenerated, never stored)
  const T* box;                   // [B,C] the forward's periodic box lengths (PBC instantiations only)
  double* g_lat;                  // dL/dbox [B,C] or dL/dcell [B,C,C] in fp64, zeroed by the caller (bwd3's LAT
                                  // instantiations only; null otherwise)
};

template <typename T> __device__ __forceinline__ T dsilu_from(T x, T sg) { return sg * (T(1) + x * (T(1) - sg)); }

// sigmoid for the bwd2 kernels: ex2.approx.ftz directly (no range fix-up: +-inf / 0 are the right limits here).
__device__ __forceinline__ float sigmoid_bw(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  return __fdividef(1.0f, 1.0f + e);
}
__device__ __forceinline__ double sigmoid_bw(double x) { return 1.0 / (1.0 + exp(-x)); }

// Record index of pair (b, i, slot).  kNN: row-major (b, i, slot).  Dense: (b, j, i) -- "column-major" -- so that the
// records of 32 consecutive rows i for one neighbour j are contiguous, which is what a bwd2 CTA streams.  Rows count
// from row0 over row1 - row0 per graph for a row block (BLK, pair_row), so its record is sized by the block.
template <bool KNN, bool BLK>
__device__ __forceinline__ size_t rec_index(const Dims& s, int b, int N, int J, int i, int slot) {
  if (!BLK) return KNN ? ((size_t)b * N + i) * J + slot : ((size_t)b * N + slot) * N + i;
  const int R = s.row1 - s.row0, r = i - s.row0;
  return KNN ? ((size_t)b * R + r) * J + slot : ((size_t)b * N + slot) * R + r;
}

// The i-rows a backward pair kernel covers: the row block (BLK), else all N rows.
template <bool BLK> __device__ __forceinline__ int rows_begin(const Dims& s) { return BLK ? s.row0 : 0; }
template <bool BLK> __device__ __forceinline__ int rows_end(const Dims& s) { return BLK ? s.row1 : s.N; }

__device__ __forceinline__ void cp_async_elem(void* smem_dst, const float* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_elem(void* smem_dst, const double* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit_group() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// =====================================================================================
// bwd1
// =====================================================================================
template <typename T>
inline size_t bwd1_smem_bytes(const Dims& s, const SimtPackLayout& L, bool soft) {
  const int U = 4 * s.m;
  size_t n = 0;
  n += (size_t)U * L.MP + 2 * U + 2 * L.MP + 4;   // w3s, b3s, w4s, misc
  n += (size_t)(soft ? 3 : 2) * PAIR_THREADS * L.MP;   // mms, gp2s, aux
  n += PAIR_THREADS;                           // gw0s
  n += (size_t)PAIR_THREADS * (U + 1);         // tt
  return round_up(n * sizeof(T), 16) + 16;
}

template <typename T, int MP, bool KNN, bool BLK, int PBC = PBC_NONE>
__global__ void __launch_bounds__(PAIR_THREADS)
pair_bwd1_kernel(const BwdArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Dims& s = a.s;
  const int tid = threadIdx.x;
  const int TS = a.TS, TI = PAIR_THREADS / TS;
  const int g = tid / TS, sl = tid % TS;
  const int b = blockIdx.y;
  T* pb = nullptr;
  if constexpr (PBC) {
    __shared__ T box_s[2 * PAIR_CMAX];
    pb = box_s;
    stage_box<T, PBC>(pb, a.box, b, s.C);
  }
  const int i_raw = rows_begin<BLK>(s) + blockIdx.x * TI + g;
  const bool row_valid = i_raw < rows_end<BLK>(s);
  const int i = row_valid ? i_raw : rows_begin<BLK>(s);
  const int J = KNN ? s.k : s.N;
  const int U = 4 * s.m, UP = U + 1;
  const bool upd_feats = a.flags & EGNN_FLAG_UPDATE_FEATS;
  const bool upd_coors = a.flags & EGNN_FLAG_UPDATE_COORS;
  const bool soft = a.flags & EGNN_FLAG_SOFT_EDGES;
  const bool normc = a.flags & EGNN_FLAG_NORM_COORS;
  const bool clampf = a.flags & EGNN_FLAG_CLAMP;

  T* w3s = reinterpret_cast<T*>(smem_raw);                 // [U][MP]
  T* b3s = w3s + U * MP;                                   // [U]
  T* w4s = b3s + U;                                        // [U]
  T* misc = w4s + U;                                       // b2[MP] | gate_w[MP] | gate_b, b4, scale, 0
  T* mms = misc + 2 * MP + 4;                              // [128][MP]  m_ij (after the gate)
  T* gp2s = mms + PAIR_THREADS * MP;                       // [128][MP]  g_pre2
  T* aux = gp2s + PAIR_THREADS * MP;                       // [128][MP]  g_z * s2 (soft edges)
  T* gw0s = aux + (soft ? PAIR_THREADS * MP : 0);          // [128]
  T* tt = gw0s + PAIR_THREADS;                             // [128][U+1] coors_mlp pre-activations

  const T* pk = a.packed;
  for (int x = tid; x < U * MP; x += PAIR_THREADS) w3s[x] = upd_coors ? pk[a.L.w3 + x] : T(0);
  for (int x = tid; x < U; x += PAIR_THREADS) {
    b3s[x] = upd_coors ? pk[a.L.b3 + x] : T(0);
    w4s[x] = upd_coors ? pk[a.L.w4 + x] : T(0);
  }
  for (int x = tid; x < 2 * MP + 4; x += PAIR_THREADS) misc[x] = pk[a.L.misc + x];
  // (visibility: the __syncthreads at the top of the pair loop)

  const size_t node_i = (size_t)b * s.N + i;
  const T* xi = a.coors + node_i * s.C;
  const bool mask_i = a.has_mask ? (a.mask[node_i] != 0) : true;
  T gxo[PAIR_CMAX];
#pragma unroll
  for (int c = 0; c < PAIR_CMAX; ++c) gxo[c] = (c < s.C) ? a.g_coors_out[node_i * s.C + c] : T(0);

  // pooling factor (egnn_pytorch.py:325-333): 1, 1/J, or 1/count of valid pairs of this row
  T inv = T(1);
  if (upd_feats && (a.flags & EGNN_FLAG_POOL_MEAN)) {
    if (a.has_mask) {
      T cnt = T(0);
      for (int s0 = 0; s0 < J; s0 += TS) {
        const int sidx = s0 + sl;
        const PairSlot ps = pair_slot<KNN>(a.nbr_idx, a.nbr_ok, s.k, node_i, sidx, row_valid && sidx < J);
        if (ps.valid && mask_i && a.mask[(size_t)b * s.N + ps.j] != 0 && ps.ok) cnt += T(1);
      }
      for (int off = TS >> 1; off > 0; off >>= 1) cnt += shfl_xor_t<T>(cnt, off);
      inv = cnt > T(0) ? T(1) / cnt : T(0);
    } else {
      inv = T(1) / T(J);
    }
  }

  // GEMM-phase role: coors_mlp.0 row u, over the pairs [p_lo, p_hi)
  const int PG = U > 0 ? PAIR_THREADS / U : 1;
  const int role_u = tid % (U > 0 ? U : 1), role_pg = tid / (U > 0 ? U : 1);
  const bool role_on = upd_coors && role_pg < PG;
  const int p_per = PAIR_THREADS / (PG > 0 ? PG : 1);
  T accW3[MP];
#pragma unroll
  for (int o = 0; o < MP; ++o) accW3[o] = T(0);
  T accb3 = T(0), accw4 = T(0);
  T acc_col_b2 = T(0), acc_col_gw = T(0);          // threads tid < MP: column sums
  T acc_gb = T(0), acc_b4 = T(0), acc_cs = T(0);   // per-thread scalars

  for (int s0 = 0; s0 < J; s0 += TS) {
    const int sidx = s0 + sl;
    const bool pair_exists = row_valid && sidx < J;
    const PairSlot ps = pair_slot<KNN>(a.nbr_idx, a.nbr_ok, s.k, node_i, sidx, pair_exists);
    const int j = ps.j;
    const bool pair_valid = ps.valid;
    const size_t pair = node_i * s.N + j;
    T rel[PAIR_CMAX];
    const T d = pair_geometry<T, PBC>(xi, a.coors + ((size_t)b * s.N + j) * s.C, s.C, rel, pb);
    if (pair_exists) {
      T* r = a.rec + rec_index<KNN, BLK>(s, b, s.N, J, i, sidx) * a.rl.R;
      const T* erow = edge_row(a.edges, KNN && (a.flags & EGNN_FLAG_EDGES_PER_SLOT), node_i, sidx, j, s.N, s.k, s.edge_dim);
      for (int q = 0; q < s.Q; ++q) r[a.rl.f + q] = pair_channel<T>(s, erow, q, d);
    }

    // ---- W2 silu(pre1) of this pair, as the forward (or its recompute) left it (empty slots were never stored: they
    // read as zeros).  An accumulator wider than 32 registers (fp64, m_dim > 16) is read again for the second SiLU
    // rather than held through the coordinate branch, where it would spill.
    constexpr bool REREAD = MP * sizeof(T) > 32 * 4;
    const T* pre2_src = a.pre2 + ((BLK ? pair_row<true>(s, b, i) : node_i) * (size_t)J + sidx) * MP;
    auto load_pre2 = [&](T (&v)[MP]) {
#pragma unroll
      for (int o = 0; o < MP; ++o) v[o] = T(0);
      if (pair_valid) {
#pragma unroll
        for (int o = 0; o < MP; o += 4) {
          Vec4<T> t;
          t.load_g(pre2_src + o);
#pragma unroll
          for (int z = 0; z < 4; ++z) v[o + z] = t.v[z];
        }
      }
    };
    T acc[MP];
    __syncthreads();                                 // shared tiles of the previous iteration fully consumed
    load_pre2(acc);

    // ---- pair epilogue, forward
    T mm[MP];
    const T gate = pair_message<T, MP>(acc, misc, a.flags, mm);      // mm = s2 * gate
    bool pm = pair_valid;
    if (a.has_mask) pm = pm && mask_i && a.mask[(size_t)b * s.N + j] != 0 && ps.ok;

    // ---- backward through the coordinate branch (egnn_pytorch.py:302-315 reversed)
    T gmm[MP];
#pragma unroll
    for (int o = 0; o < MP; ++o) gmm[o] = T(0);
    T coef = T(0), gdn = T(0), gw0 = T(0);
    if (upd_coors) {
      T w0 = misc[2 * MP + 1];
      for (int u = 0; u < U; ++u) {
        T t = b3s[u];
        const T* w3 = w3s + u * MP;
#pragma unroll
        for (int o = 0; o < MP; o += 4) {
          Vec4<T> wv;
          wv.load(w3 + o);
#pragma unroll
          for (int z = 0; z < 4; ++z) t = fma_t(wv.v[z], mm[o + z], t);
        }
        if (a.drop.thr) {                                // coors_mlp Dropout: a dropped unit is stored as NaN (silu(0) = 0
          const T f = drop_mul<T>(a.drop, 1u, (unsigned long long)pair * U + u);   // adds nothing)
          t = f == T(0) ? T(NAN) : t * f;
        }
        tt[tid * UP + u] = t;
        if (t == t) w0 = fma_t(w4s[u], silu_acc<T>(t), w0);
      }
      const T w1 = pm ? w0 : T(0);
      bool inside = true;
      T w2 = w1;
      if (clampf) {
        inside = (w1 >= -a.clamp) && (w1 <= a.clamp);
        w2 = w1 < -a.clamp ? -a.clamp : (w1 > a.clamp ? a.clamp : w1);
      }
      if (!pair_valid) w2 = T(0);
      T scale = T(1), den = T(1), nrm = T(0);
      const T cs = misc[2 * MP + 2];
      if (normc) {
        nrm = sqrt(d);
        den = nrm > T(1e-8) ? nrm : T(1e-8);
        scale = cs / den;
      }
      coef = w2 * scale;
      T gcoef = T(0);
      if (pair_valid) {
#pragma unroll
        for (int c = 0; c < PAIR_CMAX; ++c) gcoef = fma_t(gxo[c], rel[c], gcoef);
      }
      const T gw2 = gcoef * scale;
      if (normc) {
        const T gscale = gcoef * w2;
        acc_cs += gscale / den;
        const T gnrm = (nrm >= T(1e-8)) ? -gscale * cs / (den * den) : T(0);
        gdn = (nrm > T(0)) ? gnrm / (T(2) * nrm) : T(0);
      }
      gw0 = (pm && inside) ? gw2 : T(0);
      acc_b4 += gw0;
      for (int u = 0; u < U; ++u) {
        const T t = tt[tid * UP + u];
        if (t != t) continue;                            // dropped unit: no gradient
        const T sg = sigmoid_acc<T>(t);
        const T gt = gw0 * w4s[u] * dsilu_from<T>(t, sg) * (a.drop.thr ? drop_scale<T>(a.drop) : T(1));
        const T* w3 = w3s + u * MP;
#pragma unroll
        for (int o = 0; o < MP; o += 4) {
          Vec4<T> wv;
          wv.load(w3 + o);
#pragma unroll
          for (int z = 0; z < 4; ++z) gmm[o + z] = fma_t(wv.v[z], gt, gmm[o + z]);
        }
      }
    }
    gw0s[tid] = gw0;
    // ---- pooled message (egnn_pytorch.py:319-333 reversed)
    if (upd_feats && pm) {
      const T* gmi = a.g_node_in + node_i * a.ld_g + s.dim;
#pragma unroll
      for (int o = 0; o < MP; ++o)
        if (o < s.m) gmm[o] = fma_t(gmi[o], inv, gmm[o]);
    }
#pragma unroll
    for (int o = 0; o < MP; ++o) mms[tid * MP + o] = mm[o];
    // ---- gate and the second SiLU (egnn_pytorch.py:287-290 reversed); s2 and silu'(pre2) recomputed from pre2
    if (REREAD) load_pre2(acc);
    T gz = T(0);
    if (soft) {
      T ggt = T(0);
#pragma unroll
      for (int o = 0; o < MP; ++o) ggt = fma_t(gmm[o], silu_acc<T>(acc[o] + misc[o]), ggt);
      gz = ggt * gate * (T(1) - gate);
      acc_gb += gz;
    }
#pragma unroll
    for (int o = 0; o < MP; ++o) {
      const T p2 = acc[o] + misc[o];
      const T sg = sigmoid_acc<T>(p2);
      const T s2 = p2 * sg;
      T gs2 = gmm[o];
      if (soft) {
        gs2 = fma_t(gz, misc[MP + o], gmm[o] * gate);
        aux[tid * MP + o] = gz * s2;
      }
      const T gp2 = gs2 * dsilu_from<T>(p2, sg);
      gp2s[tid * MP + o] = gp2;
      gmm[o] = gp2;                                   // reuse as the value written to the record
    }
    if (pair_exists) {
      T* r = a.rec + rec_index<KNN, BLK>(s, b, s.N, J, i, sidx) * a.rl.R;
#pragma unroll
      for (int o = 0; o < MP; ++o) r[a.rl.gpre2 + o] = gmm[o];
      r[a.rl.coef] = coef;
      r[a.rl.gdn] = gdn;
    }
    __syncthreads();
    // ---- CTA-level parameter gradients of this tile of 128 pairs
    if (role_on) {
      const T w4u = w4s[role_u];
      for (int p = role_pg * p_per; p < (role_pg + 1) * p_per; ++p) {
        const T g0 = gw0s[p];
        if (g0 == T(0)) continue;
        const T t = tt[p * UP + role_u];
        if (t != t) continue;                            // dropped unit
        const T sg = sigmoid_acc<T>(t);
        const T gt = g0 * w4u * dsilu_from<T>(t, sg) * (a.drop.thr ? drop_scale<T>(a.drop) : T(1));
        accb3 += gt;
        accw4 = fma_t(g0, t * sg, accw4);
        const T* mrow = mms + p * MP;
#pragma unroll
        for (int o = 0; o < MP; o += 4) {
          Vec4<T> mv;
          mv.load(mrow + o);
#pragma unroll
          for (int z = 0; z < 4; ++z) accW3[o + z] = fma_t(gt, mv.v[z], accW3[o + z]);
        }
      }
    }
    if (tid < MP) {
      for (int p = 0; p < PAIR_THREADS; ++p) {
        acc_col_b2 += gp2s[p * MP + tid];
        if (soft) acc_col_gw += aux[p * MP + tid];
      }
    }
    // (the next iteration's first __syncthreads orders these reads before the tiles are rewritten)
  }

  // ---- flush
  T* gpk = a.gpk;
  if (role_on) {
#pragma unroll
    for (int o = 0; o < MP; ++o)
      if (o < s.m) atomic_add_t<T>(gpk + a.L.w3 + role_u * MP + o, accW3[o]);
    atomic_add_t<T>(gpk + a.L.b3 + role_u, accb3);
    atomic_add_t<T>(gpk + a.L.w4 + role_u, accw4);
  }
  if (tid < MP) {
    atomic_add_t<T>(gpk + a.L.misc + tid, acc_col_b2);
    if (soft) atomic_add_t<T>(gpk + a.L.misc + MP + tid, acc_col_gw);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    acc_gb += shfl_xor_t<T>(acc_gb, off);
    acc_b4 += shfl_xor_t<T>(acc_b4, off);
    acc_cs += shfl_xor_t<T>(acc_cs, off);
  }
  if ((tid & 31) == 0) {
    if (soft) atomic_add_t<T>(gpk + a.L.misc + 2 * MP + 0, acc_gb);
    if (upd_coors) atomic_add_t<T>(gpk + a.L.misc + 2 * MP + 1, acc_b4);
    if (normc) atomic_add_t<T>(gpk + a.L.misc + 2 * MP + 2, acc_cs);
  }
}

// =====================================================================================
// bwd2, neighbour-list form: thread = hidden channel, CTA = TI2 rows x 128 channels.  One step = up to 32 slots of
// one row: their records are contiguous (rec_index<true>) and are prefetched one step ahead with cp.async together
// with the neighbour indices; the 32 gathered B rows are loaded up front (32 independent L2 requests per thread),
// dL/dA_i is a register, dL/dB_j one fire-and-forget atomic per (pair, channel) -- the scatter is inherent to a
// neighbour list -- and dL/df_q is reduced over the channels through a [32][128] shared tile.
// =====================================================================================
constexpr int BW2_TH = 128;       // channels per CTA
constexpr int BW2_PB = 32;        // pairs per step
constexpr int BW2_MAXLAB = 16;    // label rows kept in shared memory

template <typename T>
inline size_t bwd2_knn_smem_bytes(const Dims& s, int R) {
  const int NL = s.label_dim > 0 ? s.num_labels : 0;
  size_t n = 0;
  n += (size_t)2 * s.Q * BW2_TH;            // wqs, gwqs
  n += (size_t)2 * NL * BW2_TH;             // tabs, gtabs
  n += (size_t)2 * BW2_PB * R;              // recs (double buffered)
  n += (size_t)BW2_PB * BW2_TH;             // gps
  return round_up(n * sizeof(T), 16) + 4 * BW2_PB * sizeof(int) + 16;
}

template <typename T, int MP, int QR, bool DROP, bool BLK>
__global__ void __launch_bounds__(BW2_TH)
pair_bwd2_knn_kernel(const BwdArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Dims& s = a.s;
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.z;
  const int i0 = rows_begin<BLK>(s) + blockIdx.x * a.TI2;
  const int h0 = blockIdx.y * BW2_TH;
  const int hh = h0 + tid;
  const bool hv = hh < s.Hp;
  const int N = s.N, R = a.rl.R, Q = s.Q, k = s.k;
  const int NL = s.label_dim > 0 ? s.num_labels : 0;
  const int nrows = min(a.TI2, (BLK ? s.row1 : N) - i0);
  const int nch = ceil_div(k, BW2_PB);
  const int nsteps = nrows * nch;

  T* wqs = reinterpret_cast<T*>(smem_raw);       // [Q][128]
  T* gwqs = wqs + Q * BW2_TH;                    // [Q][128]
  T* tabs = gwqs + Q * BW2_TH;                   // [NL][128]
  T* gtabs = tabs + NL * BW2_TH;                 // [NL][128]
  T* recs = gtabs + NL * BW2_TH;                 // [2][32][R]
  T* gps = recs + 2 * BW2_PB * R;                // [32][128]
  int* nb = reinterpret_cast<int*>(smem_raw + round_up((size_t)(2 * Q * BW2_TH + 2 * NL * BW2_TH + 2 * BW2_PB * R +
                                                                 BW2_PB * BW2_TH) * sizeof(T), 16));      // [2][32] neighbour
  int* lb = nb + 2 * BW2_PB;                                                                              // [2][32] label

  const T* pk = a.packed;
  for (int q = 0; q < Q; ++q) {
    wqs[q * BW2_TH + tid] = hv ? pk[a.L.wq + (size_t)q * s.Hp + hh] : T(0);
    gwqs[q * BW2_TH + tid] = T(0);
  }
  for (int l = 0; l < NL; ++l) {
    tabs[l * BW2_TH + tid] = hv ? pk[a.L.tab + (size_t)l * s.Hp + hh] : T(0);
    gtabs[l * BW2_TH + tid] = T(0);
  }
  T w2r[MP], gW2[MP];
#pragma unroll
  for (int o = 0; o < MP; ++o) {
    w2r[o] = hv ? pk[a.L.w2t + (size_t)hh * MP + o] : T(0);
    gW2[o] = T(0);
  }
  const T wq0 = hv ? pk[a.L.wq + (size_t)(2 * s.F) * s.Hp + hh] : T(0);
  T gwq0 = T(0);
  constexpr bool SIMPLE = QR == 1;          // distance channel only, no label table
  constexpr bool QREG = QR > 1;             // Q <= QR: per-pair scalar channels and their weights live in registers
  constexpr int QN = QREG ? QR : 1;
  T wqr[QN], gwqr[QN];
#pragma unroll
  for (int q = 0; q < QN; ++q) {
    wqr[q] = (QREG && q < Q && hv) ? pk[a.L.wq + (size_t)q * s.Hp + hh] : T(0);
    gwqr[q] = T(0);
  }

  auto prefetch = [&](int t, int buf) {
    const int row = t / nch, c0 = (t % nch) * BW2_PB, kc = min(BW2_PB, k - c0);
    const size_t node = (size_t)b * N + i0 + row;
    const T* src = a.rec + rec_index<true, BLK>(s, b, N, k, i0 + row, c0) * R;
    T* dst = recs + buf * BW2_PB * R;
    for (int x = tid; x < kc * R; x += BW2_TH) cp_async_elem(dst + x, src + x);
    if (tid < BW2_PB) {
      const int j = tid < kc ? a.nbr_idx[node * k + c0 + tid] : -1;
      nb[buf * BW2_PB + tid] = j;
      lb[buf * BW2_PB + tid] = (NL && j >= 0) ? a.labels[node * N + j] : 0;
    }
    cp_async_commit_group();
  };
  if (nsteps > 0) prefetch(0, 0);
  cp_async_wait_all();
  __syncthreads();

  int cur_row = -1;
  T Ai = T(0), gA = T(0);
  for (int t = 0; t < nsteps; ++t) {
    const int cur = t & 1;
    const int row = t / nch, c0 = (t % nch) * BW2_PB, kc = min(BW2_PB, k - c0);
    if (t + 1 < nsteps) prefetch(t + 1, cur ^ 1);
    if (row != cur_row) {
      if (cur_row >= 0 && hv) a.gP[((size_t)b * N + i0 + cur_row) * a.ldP + hh] = gA;
      gA = T(0);
      cur_row = row;
      Ai = hv ? a.P[((size_t)b * N + i0 + row) * a.ldP + hh] : T(0);
    }
    const int* nbc = nb + cur * BW2_PB;
    const T* rb = recs + cur * BW2_PB * R;
    T bjv[BW2_PB];
#pragma unroll
    for (int p = 0; p < BW2_PB; ++p) {
      const int j = nbc[p];
      bjv[p] = (j >= 0 && hv) ? a.P[((size_t)b * N + j) * a.ldP + s.Hp + hh] : T(0);
    }
#pragma unroll
    for (int p = 0; p < BW2_PB; ++p) {
      if (p >= kc) break;                              // uniform
      const int j = nbc[p];
      T gp = T(0);
      if (j >= 0) {                                    // uniform
        const T* r = rb + p * R;
        T pre = Ai + bjv[p];
        int lab = 0;
        T fq[QN];
        if (SIMPLE) {
          pre = fma_t(wq0, r[MP], pre);
        } else {
          if (QREG) {
#pragma unroll
            for (int q = 0; q < QN; ++q)
              if (q < Q) { fq[q] = r[MP + q]; pre = fma_t(wqr[q], fq[q], pre); }
          } else {
            for (int q = 0; q < Q; ++q) pre = fma_t(wqs[q * BW2_TH + tid], r[MP + q], pre);
          }
          if (NL) { lab = lb[cur * BW2_PB + p]; pre += tabs[lab * BW2_TH + tid]; }
        }
        T fdrop = T(1);
        if (DROP) {                                      // edge_mlp Dropout: same mask as the forward (own instantiation: the
                                                         // key arithmetic costs 50 registers when unrolled over the rows)
          fdrop = drop_mul<T>(a.drop, 0u, (((unsigned long long)b * N + i0 + row) * N + j) * s.Hp + hh);
          pre *= fdrop;
        }
        const T sg = sigmoid_bw(pre);
        const T a1 = pre * sg;
        T ga1e[2] = {T(0), T(0)};                       // even / odd channels, summed at the end
#pragma unroll
        for (int o = 0; o < MP; o += 4) {
          Vec4<T> gv;
          gv.load(r + o);
#pragma unroll
          for (int z = 0; z < 4; ++z) {
            ga1e[z & 1] = fma_t(w2r[o + z], gv.v[z], ga1e[z & 1]);
            gW2[o + z] = fma_t(a1, gv.v[z], gW2[o + z]);
          }
        }
        const T ga1 = ga1e[0] + ga1e[1];
        gp = ga1 * dsilu_from<T>(pre, sg);
        if (DROP) gp *= fdrop;
        gA += gp;
        if (hv) atomic_add_t<T>(a.gP + ((size_t)b * N + j) * a.ldP + s.Hp + hh, gp);
        if (SIMPLE) {
          gwq0 = fma_t(r[MP], gp, gwq0);
        } else {
          if (QREG) {
#pragma unroll
            for (int q = 0; q < QN; ++q)
              if (q < Q) gwqr[q] = fma_t(fq[q], gp, gwqr[q]);
          } else {
            for (int q = 0; q < Q; ++q) gwqs[q * BW2_TH + tid] = fma_t(r[MP + q], gp, gwqs[q * BW2_TH + tid]);
          }
          if (NL) gtabs[lab * BW2_TH + tid] += gp;
        }
      }
      gps[p * BW2_TH + tid] = SIMPLE ? wq0 * gp : gp;      // SIMPLE: the tile holds Wq[h] * g_pre1 already
    }
    __syncthreads();                                   // gps complete
    {
      const int p = tid >> 2, qt = tid & 3;
      const bool live = p < kc && nbc[p] >= 0;
      const T* grow = gps + p * BW2_TH + qt * 32;
      for (int q = 0; q < Q; ++q) {
        const T* wrow = wqs + q * BW2_TH + qt * 32;
        T v = T(0);
        if (live && SIMPLE) {
#pragma unroll
          for (int kx = 0; kx < 8; ++kx) {
            Vec4<T> t;
            t.load(grow + 4 * ((kx + lane) & 7));
            v += (t.v[0] + t.v[1]) + (t.v[2] + t.v[3]);
          }
        } else if (live) {
#pragma unroll 8
          for (int kx = 0; kx < 32; ++kx) {
            const int kk = (kx + lane) & 31;
            v = fma_t(wrow[kk], grow[kk], v);
          }
        }
        v += shfl_xor_t<T>(v, 1);
        v += shfl_xor_t<T>(v, 2);
        if (qt == 0 && live) atomic_add_t<T>(a.rec + rec_index<true, BLK>(s, b, N, k, i0 + row, c0 + p) * R + a.rl.gf + q, v);
      }
    }
    cp_async_wait_all();
    __syncthreads();                                   // next records landed; gps free
  }
  if (hv) {
    if (cur_row >= 0) a.gP[((size_t)b * N + i0 + cur_row) * a.ldP + hh] = gA;
#pragma unroll
    for (int o = 0; o < MP; ++o) atomic_add_t<T>(a.gpk + a.L.w2t + (size_t)hh * MP + o, gW2[o]);
    if (SIMPLE) {
      atomic_add_t<T>(a.gpk + a.L.wq + (size_t)(2 * s.F) * s.Hp + hh, gwq0);
    } else {
      if (QREG) {
#pragma unroll
        for (int q = 0; q < QN; ++q)
          if (q < Q) atomic_add_t<T>(a.gpk + a.L.wq + (size_t)q * s.Hp + hh, gwqr[q]);
      } else {
        for (int q = 0; q < Q; ++q) atomic_add_t<T>(a.gpk + a.L.wq + (size_t)q * s.Hp + hh, gwqs[q * BW2_TH + tid]);
      }
      for (int l = 0; l < NL; ++l) atomic_add_t<T>(a.gpk + a.L.tab + (size_t)l * s.Hp + hh, gtabs[l * BW2_TH + tid]);
    }
  }
}

// =====================================================================================
// bwd2, dense all-pairs specialisation: CTA = 32 rows x 128 channels, one neighbour j per step.  The 32 records of
// (i0..i0+31, j) are contiguous (rec_index<false>) and are prefetched one step ahead with cp.async; row sums dL/dA live
// in registers (the pair loop is unrolled over the 32 rows), the column sum dL/dB_j is one atomic per step, and
// dL/df_q is reduced over the 128 channels through a [32][128] shared tile instead of per-pair shuffles.
// SIMPLE = only the distance channel (Q == 1) and no label table: the common EGNN(dim) configuration.
// =====================================================================================
constexpr int BW2_ROWS = 32;

template <typename T>
inline size_t bwd2_dense_smem_bytes(const Dims& s, int R) {
  const int NL = s.label_dim > 0 ? s.num_labels : 0;
  size_t n = 0;
  n += (size_t)BW2_ROWS * BW2_TH;           // As
  n += (size_t)2 * s.Q * BW2_TH;            // wqs, gwqs
  n += (size_t)2 * NL * BW2_TH;             // tabs, gtabs
  n += (size_t)2 * BW2_ROWS * R;            // recs (double buffered)
  n += (size_t)BW2_ROWS * BW2_TH;           // gps
  return round_up(n * sizeof(T), 16) + 2 * BW2_ROWS * sizeof(int) + 16;
}

template <typename T, int MP, int QR, bool DROP, bool BLK>
__global__ void __launch_bounds__(BW2_TH)
pair_bwd2_dense_kernel(const BwdArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Dims& s = a.s;
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.z;
  const int i0 = rows_begin<BLK>(s) + blockIdx.x * BW2_ROWS;
  const int h0 = blockIdx.y * BW2_TH;
  const int hh = h0 + tid;
  const bool hv = hh < s.Hp;
  const int N = s.N, R = a.rl.R, Q = s.Q;
  const int NL = s.label_dim > 0 ? s.num_labels : 0;
  const int nrows = min(BW2_ROWS, (BLK ? s.row1 : N) - i0);

  T* As = reinterpret_cast<T*>(smem_raw);        // [32][128]
  T* wqs = As + BW2_ROWS * BW2_TH;               // [Q][128]
  T* gwqs = wqs + Q * BW2_TH;                    // [Q][128]
  T* tabs = gwqs + Q * BW2_TH;                   // [NL][128]
  T* gtabs = tabs + NL * BW2_TH;                 // [NL][128]
  T* recs = gtabs + NL * BW2_TH;                 // [2][32][R]
  T* gps = recs + 2 * BW2_ROWS * R;              // [32][128]
  int* labs = reinterpret_cast<int*>(smem_raw + round_up((size_t)(2 * BW2_ROWS * BW2_TH + 2 * Q * BW2_TH + 2 * NL * BW2_TH +
                                                                   2 * BW2_ROWS * R) * sizeof(T), 16));   // [2][32]

  const T* pk = a.packed;
  for (int r = 0; r < BW2_ROWS; ++r)
    As[r * BW2_TH + tid] = (r < nrows && hv) ? a.P[((size_t)b * N + i0 + r) * a.ldP + hh] : T(0);
  for (int q = 0; q < Q; ++q) {
    wqs[q * BW2_TH + tid] = hv ? pk[a.L.wq + (size_t)q * s.Hp + hh] : T(0);
    gwqs[q * BW2_TH + tid] = T(0);
  }
  for (int l = 0; l < NL; ++l) {
    tabs[l * BW2_TH + tid] = hv ? pk[a.L.tab + (size_t)l * s.Hp + hh] : T(0);
    gtabs[l * BW2_TH + tid] = T(0);
  }
  for (int x = tid; x < 2 * BW2_ROWS * R; x += BW2_TH) recs[x] = T(0);     // rows >= nrows stay zero
  if (tid < 2 * BW2_ROWS) labs[tid] = 0;
  T gA[BW2_ROWS];
  T w2r[MP], gW2[MP];
#pragma unroll
  for (int o = 0; o < MP; ++o) {
    w2r[o] = hv ? pk[a.L.w2t + (size_t)hh * MP + o] : T(0);
    gW2[o] = T(0);
  }
#pragma unroll
  for (int p = 0; p < BW2_ROWS; ++p) gA[p] = T(0);
  const T wq0 = hv ? pk[a.L.wq + (size_t)(2 * s.F) * s.Hp + hh] : T(0);   // SIMPLE: the distance column
  T gwq0 = T(0);
  constexpr bool SIMPLE = QR == 1;          // distance channel only, no label table
  constexpr bool QREG = QR > 1;             // Q <= QR: per-pair scalar channels and their weights live in registers
  constexpr int QN = QREG ? QR : 1;
  T wqr[QN], gwqr[QN];
#pragma unroll
  for (int q = 0; q < QN; ++q) {
    wqr[q] = (QREG && q < Q && hv) ? pk[a.L.wq + (size_t)q * s.Hp + hh] : T(0);
    gwqr[q] = T(0);
  }
  __syncthreads();

  auto prefetch = [&](int j, int buf) {
    const T* src = a.rec + rec_index<false, BLK>(s, b, N, N, i0, j) * R;
    T* dst = recs + buf * BW2_ROWS * R;
    for (int x = tid; x < nrows * R; x += BW2_TH) cp_async_elem(dst + x, src + x);
    if (!SIMPLE && NL && tid < nrows) labs[buf * BW2_ROWS + tid] = a.labels[((size_t)b * N + i0 + tid) * N + j];
    cp_async_commit_group();
  };
  prefetch(0, 0);
  T bj_next = hv ? a.P[((size_t)b * N) * a.ldP + s.Hp + hh] : T(0);
  cp_async_wait_all();
  __syncthreads();

  for (int j = 0; j < N; ++j) {
    const int cur = j & 1;
    if (j + 1 < N) prefetch(j + 1, cur ^ 1);
    const T bj = bj_next;
    if (j + 1 < N) bj_next = hv ? a.P[((size_t)b * N + j + 1) * a.ldP + s.Hp + hh] : T(0);
    const T* rb = recs + cur * BW2_ROWS * R;
    T gB = T(0);
#pragma unroll
    for (int p = 0; p < BW2_ROWS; ++p) {
      const T* r = rb + p * R;
      T pre = As[p * BW2_TH + tid] + bj;
      int lab = 0;
      T fq[QN];
      if (SIMPLE) {
        pre = fma_t(wq0, r[MP], pre);
      } else {
        if (QREG) {
#pragma unroll
          for (int q = 0; q < QN; ++q)
            if (q < Q) { fq[q] = r[MP + q]; pre = fma_t(wqr[q], fq[q], pre); }
        } else {
          for (int q = 0; q < Q; ++q) pre = fma_t(wqs[q * BW2_TH + tid], r[MP + q], pre);
        }
        if (NL) { lab = labs[cur * BW2_ROWS + p]; pre += tabs[lab * BW2_TH + tid]; }
      }
      T fdrop = T(1);
      if (DROP) {                                        // edge_mlp Dropout: same mask as the forward
        fdrop = drop_mul<T>(a.drop, 0u, (((unsigned long long)b * N + i0 + p) * N + j) * s.Hp + hh);
        pre *= fdrop;
      }
      const T sg = sigmoid_bw(pre);
      const T a1 = pre * sg;
      T ga1e[2] = {T(0), T(0)};                       // even / odd channels, summed at the end
#pragma unroll
      for (int o = 0; o < MP; o += 4) {
        Vec4<T> gv;
        gv.load(r + o);
#pragma unroll
        for (int z = 0; z < 4; ++z) {
          ga1e[z & 1] = fma_t(w2r[o + z], gv.v[z], ga1e[z & 1]);
          gW2[o + z] = fma_t(a1, gv.v[z], gW2[o + z]);
        }
      }
      const T ga1 = ga1e[0] + ga1e[1];
      T gp = ga1 * dsilu_from<T>(pre, sg);
      if (DROP) gp *= fdrop;
      gA[p] += gp;
      gB += gp;
      gps[p * BW2_TH + tid] = SIMPLE ? wq0 * gp : gp;      // SIMPLE: the tile holds Wq[h] * g_pre1 already
      if (SIMPLE) {
        gwq0 = fma_t(r[MP], gp, gwq0);
      } else {
        if (QREG) {
#pragma unroll
          for (int q = 0; q < QN; ++q)
            if (q < Q) gwqr[q] = fma_t(fq[q], gp, gwqr[q]);
        } else {
          for (int q = 0; q < Q; ++q) gwqs[q * BW2_TH + tid] = fma_t(r[MP + q], gp, gwqs[q * BW2_TH + tid]);
        }
        if (NL) gtabs[lab * BW2_TH + tid] += gp;
      }
    }
    if (hv) atomic_add_t<T>(a.gP + ((size_t)b * N + j) * a.ldP + s.Hp + hh, gB);
    __syncthreads();                                   // gps complete
    {
      // dL/df_q(i0+p, j) = sum_h Wq[q][h] gp[p][h]: thread = (row p, quarter of the channels); lanes start at
      // rotated offsets so that the 32 lanes of a warp hit 32 different banks
      const int p = tid >> 2, qt = tid & 3;
      const T* grow = gps + p * BW2_TH + qt * 32;
      for (int q = 0; q < Q; ++q) {
        const T* wrow = wqs + q * BW2_TH + qt * 32;
        T v = T(0);
        if (SIMPLE) {                                   // plain row sum, 4 values per load, rotated start per lane
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            Vec4<T> t;
            t.load(grow + 4 * ((k + lane) & 7));
            v += (t.v[0] + t.v[1]) + (t.v[2] + t.v[3]);
          }
        } else {
#pragma unroll 8
          for (int k = 0; k < 32; ++k) {
            const int kk = (k + lane) & 31;
            v = fma_t(wrow[kk], grow[kk], v);
          }
        }
        v += shfl_xor_t<T>(v, 1);
        v += shfl_xor_t<T>(v, 2);
        if (qt == 0 && p < nrows) atomic_add_t<T>(a.rec + rec_index<false, BLK>(s, b, N, N, i0 + p, j) * R + a.rl.gf + q, v);
      }
    }
    cp_async_wait_all();
    __syncthreads();                                   // next records landed; gps free
  }
  if (hv) {
#pragma unroll
    for (int p = 0; p < BW2_ROWS; ++p)
      if (p < nrows) a.gP[((size_t)b * N + i0 + p) * a.ldP + hh] = gA[p];
#pragma unroll
    for (int o = 0; o < MP; ++o) atomic_add_t<T>(a.gpk + a.L.w2t + (size_t)hh * MP + o, gW2[o]);
    if (SIMPLE) {
      atomic_add_t<T>(a.gpk + a.L.wq + (size_t)(2 * s.F) * s.Hp + hh, gwq0);
    } else {
      if (QREG) {
#pragma unroll
        for (int q = 0; q < QN; ++q)
          if (q < Q) atomic_add_t<T>(a.gpk + a.L.wq + (size_t)q * s.Hp + hh, gwqr[q]);
      } else {
        for (int q = 0; q < Q; ++q) atomic_add_t<T>(a.gpk + a.L.wq + (size_t)q * s.Hp + hh, gwqs[q * BW2_TH + tid]);
      }
      for (int l = 0; l < NL; ++l) atomic_add_t<T>(a.gpk + a.L.tab + (size_t)l * s.Hp + hh, gtabs[l * BW2_TH + tid]);
    }
  }
}

// =====================================================================================
// bwd3: dL/d(dist) -> coordinates and edges.  Same thread <-> pair mapping as bwd1.  PBC: the minimum image has the
// derivative of x_i - x_j (rint is piecewise constant), so only rel changes.
// LAT (PBC instantiations only): also the lattice gradient.  rel = (x_i - x_j) - sum_c n_c a_c with integer image
// counts n, so with gr = dL/d rel:  dL/dcell[c][d] = -sum_pairs n_c gr_d (d <= c),  dL/dbox[c] = -sum_pairs n_c gr_c.
// Each thread sums its pairs in fp64 (either T); the sums are reduced over the warp, then over the CTA's warps in
// shared memory, and the CTA (one graph, blockIdx.y) adds them to g_lat[b] with one atomicAdd per entry.
// =====================================================================================
// Lattice entries a bwd3 thread accumulates: the lower triangle of a cell (00, 10, 11, 20, 21, 22) or every box axis.
template <int PBC> __host__ __device__ constexpr int lat_entries() { return PBC == PBC_CELL ? 6 : PAIR_CMAX; }
__host__ __device__ constexpr int lat_row(int e) { return e == 0 ? 0 : e < 3 ? 1 : 2; }
__host__ __device__ constexpr int lat_col(int e) { return e == 0 ? 0 : e < 3 ? e - 1 : e - 3; }

template <typename T, bool KNN, bool BLK, int PBC = PBC_NONE, bool LAT = false>
__global__ void __launch_bounds__(PAIR_THREADS)
pair_bwd3_kernel(const BwdArgs<T> a) {
  static_assert(!LAT || PBC != PBC_NONE, "the lattice gradient needs a box or a cell");
  const Dims& s = a.s;
  const int tid = threadIdx.x;
  const int TS = a.TS, TI = PAIR_THREADS / TS;
  const int g = tid / TS, sl = tid % TS;
  const int b = blockIdx.y;
  T* pb = nullptr;
  if constexpr (PBC) {
    __shared__ T box_s[2 * PAIR_CMAX];
    pb = box_s;
    stage_box<T, PBC>(pb, a.box, b, s.C);
  }
  const int i_raw = rows_begin<BLK>(s) + blockIdx.x * TI + g;
  const bool row_valid = i_raw < rows_end<BLK>(s);
  const int i = row_valid ? i_raw : rows_begin<BLK>(s);
  const int J = KNN ? s.k : s.N;
  const int qd = 2 * s.F;
  const size_t node_i = (size_t)b * s.N + i;
  const T* xi = a.coors + node_i * s.C;
  T gxo[PAIR_CMAX], gxi[PAIR_CMAX];
#pragma unroll
  for (int c = 0; c < PAIR_CMAX; ++c) {
    gxo[c] = (c < s.C) ? a.g_coors_out[node_i * s.C + c] : T(0);
    gxi[c] = T(0);
  }
  const bool per_slot = KNN && (a.flags & EGNN_FLAG_EDGES_PER_SLOT);
  constexpr int NL = LAT ? lat_entries<PBC>() : 1;
  double lat[NL];
#pragma unroll
  for (int e = 0; e < NL; ++e) lat[e] = 0.0;
  for (int s0 = 0; s0 < J; s0 += TS) {
    const int sidx = s0 + sl;
    const PairSlot ps = pair_slot<KNN>(a.nbr_idx, nullptr, s.k, node_i, sidx, row_valid && sidx < J);
    if (!ps.valid) continue;
    const int j = ps.j;
    const T* r = a.rec + rec_index<KNN, BLK>(s, b, s.N, J, i, sidx) * a.rl.R;
    T rel[PAIR_CMAX], nimg[PAIR_CMAX];
    const T* xj = a.coors + ((size_t)b * s.N + j) * s.C;
    T d;
    if constexpr (LAT) d = pair_geometry<T, PBC>(xi, xj, s.C, rel, nimg, pb);
    else d = pair_geometry<T, PBC>(xi, xj, s.C, rel, pb);
    T gd = r[a.rl.gf + qd] + r[a.rl.gdn];
    for (int q = 0; q < s.F; ++q) {                        // fourier_encode_dist :34-41 reversed
      const T sc = T(1 << q);
      gd += (r[a.rl.gf + q] * cos(d / sc) - r[a.rl.gf + s.F + q] * sin(d / sc)) / sc;
    }
    if (a.g_edges) {      // per-slot edges: this thread alone owns the slot, so a plain store, no atomic
      T* ge = edge_row(a.g_edges, per_slot, node_i, sidx, j, s.N, s.k, s.edge_dim);
      for (int e = 0; e < s.edge_dim; ++e) {
        if (KNN && !per_slot) atomic_add_t<T>(ge + e, r[a.rl.gf + s.Qd + e]);
        else ge[e] = r[a.rl.gf + s.Qd + e];
      }
    }
    if (j == i) continue;        // x_i - x_i: the two contributions cancel exactly (and would be 1/eps-sized under CoorsNorm)
    const T coef = r[a.rl.coef];
    T* gxj = a.g_coors + ((size_t)b * s.N + j) * s.C;
    T grv[PAIR_CMAX];
#pragma unroll
    for (int c = 0; c < PAIR_CMAX; ++c) {
      if constexpr (LAT) grv[c] = T(0);
      if (c < s.C) {
        const T gr = fma_t(coef, gxo[c], T(2) * gd * rel[c]);
        gxi[c] += gr;
        atomic_add_t<T>(gxj + c, -gr);
        if constexpr (LAT) grv[c] = gr;
      }
    }
    if constexpr (LAT) {        // n is 0 on aperiodic axes and beyond C, and gr is 0 beyond C
#pragma unroll
      for (int e = 0; e < NL; ++e) {
        const int rr = PBC == PBC_CELL ? lat_row(e) : e, cc = PBC == PBC_CELL ? lat_col(e) : e;
        lat[e] = fma(-(double)nimg[rr], (double)grv[cc], lat[e]);
      }
    }
  }
  for (int off = TS >> 1; off > 0; off >>= 1) {
#pragma unroll
    for (int c = 0; c < PAIR_CMAX; ++c) gxi[c] += shfl_xor_t<T>(gxi[c], off);
  }
  if (sl == 0 && row_valid) {
#pragma unroll
    for (int c = 0; c < PAIR_CMAX; ++c)
      if (c < s.C) atomic_add_t<T>(a.g_coors + node_i * s.C + c, gxi[c]);
  }
  if constexpr (LAT) {
    __shared__ double lat_s[PAIR_THREADS / 32][NL];
    const int lane = tid % 32, warp = tid / 32;
#pragma unroll
    for (int e = 0; e < NL; ++e) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) lat[e] += shfl_xor_t<double>(lat[e], off);
      if (lane == 0) lat_s[warp][e] = lat[e];
    }
    __syncthreads();
    if (tid < NL) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < PAIR_THREADS / 32; ++w) t += lat_s[w][tid];
      if (PBC == PBC_CELL) {
        const int rr = lat_row(tid), cc = lat_col(tid);
        if (rr < s.C) atomicAdd(a.g_lat + ((size_t)b * s.C + rr) * s.C + cc, t);
      } else if (tid < s.C) {
        atomicAdd(a.g_lat + (size_t)b * s.C + tid, t);
      }
    }
  }
}

// =====================================================================================
// Per-node pieces
// =====================================================================================
// Node rows of a row block (EGNN_FLAG_ROW_PARTIAL_GRADS) are addressed through a RowMap by the per-node backward
// kernels; ACC_PLAIN keeps the plain row index (every row, in order).  For gemm_acc_kernel the map applies to the output
// rows r of A and C (ACC_ROWS) or to the reduction index k of A and B (ACC_K).
constexpr int ACC_PLAIN = 0, ACC_ROWS = 1, ACC_K = 2;

// C[r, c] += sum_k A(r, k) B(k, c),  A(r,k) = A[r*ars + k*aks],  B(k,c) = B[k*bks + c*bcs]; K split over gridDim.z.
// Always accumulates with atomics: the caller zero-fills C or wants the sum.
template <typename T, int MAP>
__global__ void __launch_bounds__(256)
gemm_acc_kernel(const T* __restrict__ A, long ars, long aks, const T* __restrict__ Bm, long bks, long bcs,
                T* __restrict__ Cm, long ldc, int Mr, int Nc, int K, int kper, RowMap map) {
  __shared__ T As[16][64 + 4];
  __shared__ T Bs[16][64 + 4];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int kbeg = blockIdx.z * kper, kend = min(K, kbeg + kper);
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);
  const bool a_rows_fast = ars == 1, b_cols_fast = bcs == 1;
  for (int k0 = kbeg; k0 < kend; k0 += 16) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + r * 256;
      {
        const int row = a_rows_fast ? idx % 64 : idx / 16, kk = a_rows_fast ? idx / 64 : idx % 16;
        T v = T(0);
        if (m0 + row < Mr && k0 + kk < kend) {
          const long ar = MAP == ACC_ROWS ? (long)map(m0 + row) : (long)(m0 + row);
          const long ak = MAP == ACC_K ? (long)map(k0 + kk) : (long)(k0 + kk);
          v = A[ar * ars + ak * aks];
        }
        As[kk][row] = v;
      }
      {
        const int col = b_cols_fast ? idx % 64 : idx / 16, kk = b_cols_fast ? idx / 64 : idx % 16;
        T v = T(0);
        if (n0 + col < Nc && k0 + kk < kend) {
          const long bk = MAP == ACC_K ? (long)map(k0 + kk) : (long)(k0 + kk);
          v = Bm[bk * bks + (long)(n0 + col) * bcs];
        }
        Bs[kk][col] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      T av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[kk][ty * 4 + i]; bv[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma_t(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = m0 + ty * 4 + i;
    if (r >= Mr) continue;
    const long rr = MAP == ACC_ROWS ? (long)map(r) : (long)r;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = n0 + tx * 4 + j;
      if (c < Nc) atomic_add_t<T>(Cm + rr * ldc + c, acc[i][j]);
    }
  }
}

// out[c] += sum_r X[row(r)*ld + c], row(r) = map(r) when MAP, else r
template <typename T, bool MAP>
__global__ void colsum_acc_kernel(const T* __restrict__ X, long ld, int rows, int cols, T* __restrict__ out, RowMap map) {
  __shared__ T part[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  T s = T(0);
  if (c < cols)
    for (int r = blockIdx.y * 8 + threadIdx.y; r < rows; r += gridDim.y * 8) s += X[(MAP ? (long)map(r) : (long)r) * ld + c];
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    T t = T(0);
#pragma unroll
    for (int y = 0; y < 8; ++y) t += part[y][threadIdx.x];
    atomic_add_t<T>(out + c, t);
  }
}

// g[e] = g[e] * silu'(drop(pre[e])) * drop'   (node_mlp: Linear -> Dropout -> SiLU, egnn_pytorch.py:197-199; e = row * cols + col
// is the element index the forward GEMM epilogue hashed).  Element x of the n = rows * cols walked is e = x, or with MAP
// the element of row map(x / cols).
template <typename T, bool MAP>
__global__ void dsilu_mul_kernel(T* __restrict__ g, const T* __restrict__ pre, size_t n, int cols, RowMap map, DropCfg drop) {
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += (size_t)gridDim.x * blockDim.x) {
    const size_t e = MAP ? map((int)(x / cols)) * cols + x % cols : x;
    T p = pre[e], f = T(1);
    if (drop.thr) { f = drop_mul<T>(drop, 2u, (unsigned long long)e); p *= f; }
    g[e] *= dsilu_from<T>(p, sigmoid_acc<T>(p)) * f;
  }
}

// LayerNorm backward (or identity) of the first `dim` columns of g_node_in, one warp per row (row map(r) with MAP):
//   g_feats[row] += d(node_norm)/dh . g_normed;  gyx[row] = g_normed * xhat  (for dL/dgamma by column sum)
template <typename T, bool MAP>
__global__ void ln_bwd_kernel(const T* __restrict__ h, const T* __restrict__ gamma, const T* __restrict__ g_node_in,
                              int ld_g, T* __restrict__ g_feats, T* __restrict__ gyx, int dim, int M, int do_norm, RowMap map) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (r >= M) return;
  const size_t row = MAP ? map(r) : (size_t)r;
  const T* x = h + (size_t)row * dim;
  const T* gy = g_node_in + (size_t)row * ld_g;
  T* go = g_feats + (size_t)row * dim;
  if (!do_norm) {
    for (int c = lane; c < dim; c += 32) go[c] += gy[c];
    return;
  }
  T sm = T(0);
  for (int c = lane; c < dim; c += 32) sm += x[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sm += shfl_xor_t<T>(sm, o);
  const T mu = sm / T(dim);
  T v = T(0);
  for (int c = lane; c < dim; c += 32) { const T t = x[c] - mu; v += t * t; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += shfl_xor_t<T>(v, o);
  const T rstd = T(1) / sqrt(v / T(dim) + T(1e-5));
  T m1 = T(0), m2 = T(0);
  for (int c = lane; c < dim; c += 32) {
    const T xh = (x[c] - mu) * rstd, gg = gy[c] * gamma[c];
    m1 += gg;
    m2 += gg * xh;
    gyx[(size_t)row * dim + c] = gy[c] * xh;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { m1 += shfl_xor_t<T>(m1, o); m2 += shfl_xor_t<T>(m2, o); }
  m1 /= T(dim);
  m2 /= T(dim);
  for (int c = lane; c < dim; c += 32) {
    const T xh = (x[c] - mu) * rstd, gg = gy[c] * gamma[c];
    go[c] += rstd * (gg - m1 - xh * m2);
  }
}

// Accumulators in SimtPackLayout order -> gradients shaped like the parameters (all targets zero-filled before).
template <typename T>
__global__ void unpack_grads_kernel(Dims s, SimtPackLayout L, uint32_t flags, const T* __restrict__ gpk,
                                    const T* __restrict__ W1, const T* __restrict__ emb, EgnnLayerWeightGrads g) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int MP = L.MP, U = 4 * s.m;
  T* gW1 = static_cast<T*>((g.edge_w1));
  T* gW2 = static_cast<T*>((g.edge_w2));
  for (size_t x = t0; x < (size_t)s.m * s.H; x += stride) {
    const int o = (int)(x / s.H), c = (int)(x % s.H);
    gW2[x] = gpk[L.w2t + (size_t)c * MP + o];
  }
  for (size_t x = t0; x < (size_t)s.Q * s.H; x += stride) {
    const int q = (int)(x / s.H), c = (int)(x % s.H);
    gW1[(size_t)c * s.E + 2 * s.dim + q] = gpk[L.wq + (size_t)q * s.Hp + c];
  }
  if (s.label_dim > 0) {
    T* gemb = static_cast<T*>((g.label_emb));
    for (size_t x = t0; x < (size_t)s.label_dim * s.H; x += stride) {     // dL/dW1[c, label col a] = sum_l gTab[l,c] emb[l,a]
      const int a_ = (int)(x / s.H), c = (int)(x % s.H);
      T acc = T(0);
      for (int l = 0; l < s.num_labels; ++l) acc += gpk[L.tab + (size_t)l * s.Hp + c] * emb[(size_t)l * s.label_dim + a_];
      gW1[(size_t)c * s.E + 2 * s.dim + s.Q + a_] = acc;
    }
    if (gemb)
      for (size_t x = t0; x < (size_t)s.num_labels * s.label_dim; x += stride) {
        const int l = (int)(x / s.label_dim), a_ = (int)(x % s.label_dim);
        T acc = T(0);
        for (int c = 0; c < s.H; ++c) acc += gpk[L.tab + (size_t)l * s.Hp + c] * W1[(size_t)c * s.E + 2 * s.dim + s.Q + a_];
        gemb[x] = acc;
      }
  }
  T* gb2 = static_cast<T*>((g.edge_b2));
  for (size_t x = t0; x < (size_t)s.m; x += stride) gb2[x] = gpk[L.misc + x];
  if (flags & EGNN_FLAG_SOFT_EDGES) {
    T* ggw = static_cast<T*>((g.gate_w));
    for (size_t x = t0; x < (size_t)s.m; x += stride) ggw[x] = gpk[L.misc + MP + x];
    if (t0 == 0) static_cast<T*>((g.gate_b))[0] = gpk[L.misc + 2 * MP + 0];
  }
  if (flags & EGNN_FLAG_UPDATE_COORS) {
    T* gW3 = static_cast<T*>((g.coors_w1));
    T* gb3 = static_cast<T*>((g.coors_b1));
    T* gW4 = static_cast<T*>((g.coors_w2));
    for (size_t x = t0; x < (size_t)U * s.m; x += stride) {
      const int u = (int)(x / s.m), o = (int)(x % s.m);
      gW3[x] = gpk[L.w3 + (size_t)u * MP + o];
    }
    for (size_t x = t0; x < (size_t)U; x += stride) { gb3[x] = gpk[L.b3 + x]; gW4[x] = gpk[L.w4 + x]; }
    if (t0 == 0) static_cast<T*>((g.coors_b2))[0] = gpk[L.misc + 2 * MP + 1];
    if ((flags & EGNN_FLAG_NORM_COORS) && t0 == 0)
      static_cast<T*>((g.coors_scale))[0] = gpk[L.misc + 2 * MP + 2];
  }
}

}  // namespace egnn

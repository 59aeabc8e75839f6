// SIMT ("accurate") kernels of the EGNN layer, templated on the scalar type T (float / double).
//
// The layer is evaluated in the split form of SURVEY.md section 0:
//   W1 [h_i | h_j | d | e] + b1  =  A_i + B_j + sum_q f_q(i,j) Wq[:,q] + Tab[label(i,j)]
// with per-node tables A = h W1[:, :dim]^T + b1 and B = h W1[:, dim:2dim]^T (one GEMM each),
// so the per-pair work is H adds/FMAs + H SiLUs + the H->m contraction with W2, and nothing of
// size O(N^2 * H) is ever stored (reference egnn_pytorch.py:274-287 materialises it).
#pragma once

#include "common.cuh"

namespace egnn {

// =====================================================================================
// Parameter packing (reference layouts -> kernel layouts), see SimtPackLayout.
// =====================================================================================
template <typename T>
__global__ void simt_pack_kernel(Dims s, SimtPackLayout L, EgnnLayerWeights w, uint32_t flags, T* __restrict__ out) {
  const T* W1 = static_cast<const T*>(w.edge_w1);
  const T* W2 = static_cast<const T*>(w.edge_w2);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int MP = L.MP;
  // W2T [Hp][MP]
  for (size_t i = t0; i < (size_t)s.Hp * MP; i += stride) {
    int c = (int)(i / MP), o = (int)(i % MP);
    out[L.w2t + i] = (c < s.H && o < s.m) ? W2[(size_t)o * s.H + c] : T(0);
  }
  // Wq [Q][Hp]: columns 2dim .. 2dim+Q of W1 (distance features, then continuous edges)
  for (size_t i = t0; i < (size_t)s.Q * s.Hp; i += stride) {
    int q = (int)(i / s.Hp), c = (int)(i % s.Hp);
    out[L.wq + i] = (c < s.H) ? W1[(size_t)c * s.E + 2 * s.dim + q] : T(0);
  }
  // Tab [num_labels][Hp] = label_emb @ W1[:, label cols]^T   (egnn_pytorch.py:430-432 folded)
  if (s.label_dim > 0) {
    const T* emb = static_cast<const T*>(w.label_emb);
    for (size_t i = t0; i < (size_t)s.num_labels * s.Hp; i += stride) {
      int l = (int)(i / s.Hp), c = (int)(i % s.Hp);
      T acc = T(0);
      if (c < s.H)
        for (int a = 0; a < s.label_dim; ++a)
          acc += emb[(size_t)l * s.label_dim + a] * W1[(size_t)c * s.E + 2 * s.dim + s.Q + a];
      out[L.tab + i] = acc;
    }
  }
  const bool upd_coors = flags & EGNN_FLAG_UPDATE_COORS;
  const int U = 4 * s.m;
  if (upd_coors) {
    const T* W3 = static_cast<const T*>(w.coors_w1);
    const T* b3 = static_cast<const T*>(w.coors_b1);
    const T* W4 = static_cast<const T*>(w.coors_w2);
    for (size_t i = t0; i < (size_t)U * MP; i += stride) {
      int u = (int)(i / MP), o = (int)(i % MP);
      out[L.w3 + i] = (o < s.m) ? W3[(size_t)u * s.m + o] : T(0);
    }
    for (size_t i = t0; i < (size_t)U; i += stride) { out[L.b3 + i] = b3[i]; out[L.w4 + i] = W4[i]; }
  }
  // misc: b2[MP] | gate_w[MP] | gate_b | b4 | coors_scale | 0
  const T* b2 = static_cast<const T*>(w.edge_b2);
  for (size_t i = t0; i < (size_t)MP; i += stride) {
    out[L.misc + i] = (i < (size_t)s.m) ? b2[i] : T(0);
    T g = T(0);
    if ((flags & EGNN_FLAG_SOFT_EDGES) && i < (size_t)s.m) g = static_cast<const T*>(w.gate_w)[i];
    out[L.misc + MP + i] = g;
  }
  if (t0 == 0) {
    out[L.misc + 2 * MP + 0] = (flags & EGNN_FLAG_SOFT_EDGES) ? static_cast<const T*>(w.gate_b)[0] : T(0);
    out[L.misc + 2 * MP + 1] = upd_coors ? static_cast<const T*>(w.coors_b2)[0] : T(0);
    out[L.misc + 2 * MP + 2] = (flags & EGNN_FLAG_NORM_COORS) ? static_cast<const T*>(w.coors_scale)[0] : T(1);
    out[L.misc + 2 * MP + 3] = T(0);
  }
}

// =====================================================================================
// C[r, n] = act( sum_k A[r, k] W[n, k] + bias[n] ) (+ R[r, n]);  columns n >= Nv are written 0.
// Rows r = 0..Mr-1 map to tensor rows (r / Rr) * N + row0 + (r % Rr)  (row-range support).
// 64x64x16 tiles, 256 threads, 4x4 register tile.
// =====================================================================================
struct RowMap {
  int Rr, N, row0;
  __device__ __forceinline__ size_t operator()(int r) const { return (size_t)(r / Rr) * N + row0 + (r % Rr); }
};

template <typename T, int ACT /*0 none, 1 silu, 2 gelu (exact, erf)*/, bool RES>
__global__ void __launch_bounds__(256)
gemm_nt_kernel(const T* __restrict__ A, int lda, const T* __restrict__ W, int ldw,
               const T* __restrict__ bias, const T* __restrict__ R, int ldr,
               T* __restrict__ Cout, int ldo, int Mr, int Nv, int Nout, int K, RowMap map, DropCfg drop) {
  __shared__ T As[16][64 + 4];
  __shared__ T Ws[16][64 + 4];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);

  for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int idx = tid + r * 256;
      int row = idx / 16, kk = idx % 16;
      T av = T(0), wv = T(0);
      if (m0 + row < Mr && k0 + kk < K) av = A[map(m0 + row) * lda + k0 + kk];
      if (n0 + row < Nv && k0 + kk < K) wv = W[(size_t)(n0 + row) * ldw + k0 + kk];
      As[kk][row] = av;
      Ws[kk][row] = wv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      T a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; w[i] = Ws[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma_t(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int r = m0 + ty * 4 + i;
    if (r >= Mr) continue;
    size_t row = map(r);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int col = n0 + tx * 4 + j;
      if (col >= Nout) continue;
      T v = T(0);
      if (col < Nv) {
        v = acc[i][j] + (bias ? bias[col] : T(0));
        if (ACT == 1 && drop.thr) v *= (T)drop_mul(drop, 2u, (unsigned long long)row * Nout + col);     // node_mlp Dropout, :198
        if (ACT == 1) v = silu_acc<T>(v);
        if (ACT == 2) v = gelu_acc<T>(v);
        if (RES) v += R[row * ldr + col];
      }
      Cout[row * ldo + col] = v;
    }
  }
}

// =====================================================================================
// Same contract as gemm_nt_kernel for few rows (Mr <= 16, the latency-bound configs c1/README example):
// one warp per output column n reads W[n, :] once, coalesced, and keeps all Mr row sums in registers.
// =====================================================================================
// The latency-bound configs (BASELINE c1: 16 nodes, 12.7 MB of fp32 weights) are bound by how fast the WEIGHTS stream
// from L2 / HBM: one CTA = 4 warps x COLS output columns, the <= 16 activation rows staged once in shared memory, every
// lane pulls 16-byte pieces of its COLS weight rows (COLS independent 128-bit loads in flight per step) and keeps the
// 16 x COLS partial sums in registers; COLS is picked by the launcher so that the grid fills the SMs of the device.
constexpr int SKINNY_WARPS = 4;

template <typename T> struct SkinnyVec;            // 16-byte vector of T
template <> struct SkinnyVec<float> { static constexpr int N = 4; };
template <> struct SkinnyVec<double> { static constexpr int N = 2; };

template <typename T, int ACT, bool RES, int COLS>
__global__ void __launch_bounds__(SKINNY_WARPS * 32)
gemm_skinny_kernel(const T* __restrict__ A, int lda, const T* __restrict__ W, int ldw,
                   const T* __restrict__ bias, const T* __restrict__ R, int ldr,
                   T* __restrict__ Cout, int ldo, int Mr, int Nv, int Nout, int K, RowMap map, DropCfg drop) {
  extern __shared__ __align__(16) unsigned char skinny_smem[];
  T* As = reinterpret_cast<T*>(skinny_smem);                     // [16][Kp], Kp = K rounded up to the vector width
  constexpr int V = SkinnyVec<T>::N;
  const int Kp = (K + V - 1) / V * V;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  // staging: warp w copies rows 4w .. 4w+3; 8 independent loads in flight per lane (a dependent load -> store chain
  // per element cost 17 us of exposed L2 latency in the first version)
#pragma unroll
  for (int mm = 0; mm < 16 / SKINNY_WARPS; ++mm) {
    const int m = warp * (16 / SKINNY_WARPS) + mm;
    const T* src = A + map(m < Mr ? m : 0) * lda;
#pragma unroll 8
    for (int k = lane; k < Kp; k += 32) As[m * Kp + k] = (m < Mr && k < K) ? __ldg(src + k) : T(0);
  }
  __syncthreads();
  const int col0 = (blockIdx.x * SKINNY_WARPS + warp) * COLS;
  if (col0 >= Nout) return;
  T acc[16][COLS];
#pragma unroll
  for (int m = 0; m < 16; ++m)
#pragma unroll
    for (int n = 0; n < COLS; ++n) acc[m][n] = T(0);
  const T* wrow[COLS];
#pragma unroll
  for (int n = 0; n < COLS; ++n) wrow[n] = W + (size_t)min(col0 + n, Nv - 1) * ldw;
  // nn.Linear rows are not 16-byte aligned in general (edge_mlp.0.weight has 2*dim + 1 + ... columns), so the weight
  // rows are read with lane-strided 4-byte (8-byte for fp64) loads: fully coalesced, V independent loads per column
  // and step in flight; the staged activations are read with the same lane-strided pattern (conflict-free).
  for (int k0 = 0; k0 < Kp; k0 += 32 * V) {
    T wv[COLS][V];
#pragma unroll
    for (int n = 0; n < COLS; ++n)
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int k = k0 + v * 32 + lane;
        wv[n][v] = k < K ? __ldg(wrow[n] + k) : T(0);
      }
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      T av[V];
#pragma unroll
      for (int v = 0; v < V; ++v) { const int k = k0 + v * 32 + lane; av[v] = k < Kp ? As[m * Kp + k] : T(0); }
#pragma unroll
      for (int n = 0; n < COLS; ++n)
#pragma unroll
        for (int v = 0; v < V; ++v) acc[m][n] = fma_t(av[v], wv[n][v], acc[m][n]);
    }
  }
#pragma unroll
  for (int m = 0; m < 16; ++m)
#pragma unroll
    for (int n = 0; n < COLS; ++n)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[m][n] += shfl_xor_t<T>(acc[m][n], o);
  // every lane now holds all sums; lane l writes result number l, l + 32, ...
#pragma unroll
  for (int pass = 0; pass < (16 * COLS + 31) / 32; ++pass) {
    const int idx = pass * 32 + lane;
    const int m = idx / COLS, n = idx % COLS;
    T v = T(0);
#pragma unroll
    for (int mm = 0; mm < 16; ++mm)
#pragma unroll
      for (int nn = 0; nn < COLS; ++nn)
        if (mm == m && nn == n) v = acc[mm][nn];
    const int col = col0 + n;
    if (idx < 16 * COLS && m < Mr && col < Nout) {
      const size_t row = map(m);
      if (col < Nv) {
        v += bias ? bias[col] : T(0);
        if (ACT == 1 && drop.thr) v *= (T)drop_mul(drop, 2u, (unsigned long long)row * Nout + col);
        if (ACT == 1) v = silu_acc<T>(v);
        if (ACT == 2) v = gelu_acc<T>(v);
        if (RES) v += R[row * ldr + col];
      } else {
        v = T(0);
      }
      Cout[row * ldo + col] = v;
    }
  }
}

// =====================================================================================
// node_in[row, 0:dim] = LayerNorm(h[row]) or h[row]   (egnn_pytorch.py:335); one warp per row.
// =====================================================================================
template <typename T>
__global__ void ln_concat_kernel(const T* __restrict__ h, const T* __restrict__ g, const T* __restrict__ bta,
                                 T* __restrict__ node_in, int ld, int dim, int Mr, RowMap map, int do_norm) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (warp >= Mr) return;
  const size_t row = map(warp);
  const T* x = h + row * dim;
  T* y = node_in + row * ld;
  if (!do_norm) {
    for (int c = lane; c < dim; c += 32) y[c] = x[c];
    return;
  }
  T s = T(0);
  for (int c = lane; c < dim; c += 32) s += x[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += shfl_xor_t<T>(s, o);
  const T mu = s / T(dim);
  T v = T(0);
  for (int c = lane; c < dim; c += 32) { T t = x[c] - mu; v += t * t; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += shfl_xor_t<T>(v, o);
  const T rstd = T(1) / sqrt(v / T(dim) + T(1e-5));
  for (int c = lane; c < dim; c += 32) y[c] = (x[c] - mu) * rstd * g[c] + bta[c];
}

// =====================================================================================
// The fused edge step (reference egnn_pytorch.py:232-233, 270-333): one thread per (i, slot)
// pair, 128 threads per CTA arranged as TI row-groups x TS slots (TS lanes of one warp).
// =====================================================================================
constexpr int PAIR_THREADS = 128;
constexpr int PAIR_CH = 64;     // hidden-axis chunk staged in shared memory
constexpr int PAIR_CMAX = 8;    // max coordinate dimension

template <typename T>
struct PairArgs {
  Dims s;
  SimtPackLayout L;
  uint32_t flags;
  int has_mask;
  int TS;                    // slots per row group: 32 (dense) or pow2 >= min(k,32)
  T clamp;
  const T* P; int ldP;       // [M][2*Hp]: A | B
  const T* coors;            // [B,N,C]
  const T* edges;            // [B,N,N,edge_dim] | null
  const uint8_t* labels;     // [B,N,N] | null
  const uint8_t* mask;       // [B,N] | null
  const int32_t* nbr_idx;    // [B,N,k] (KNN)
  const uint8_t* nbr_ok;     // [B,N,k] (KNN)
  const T* packed;
  T* m_out; int ld_m;        // node_in + dim  (null when !update_feats)
  T* coors_out;              // [B,N,C]       (null when !update_coors)
  // tiny graphs only (pair_dense_tiled_kernel): the hidden axis is split over gridDim.z CTAs in phase 1, which
  // store partial m_pre sums to hpart [hsplit][B][N][N][MP]; phase 2 adds them up in a fixed order and finishes.
  T* hpart; int hsplit; int phase;      // phase 0 = single pass
  T* pre2_out;                          // optional: [B,N,J][MP] W2 silu(pre1) per pair (J = N dense, k lists), kept for backward
  DropCfg drop;                         // training-mode dropout of edge_mlp / coors_mlp hidden pre-activations (thr 0 = off)
};

template <typename T>
inline size_t pair_smem_bytes(const Dims& s, const SimtPackLayout& L, bool knn) {
  size_t n = 0;
  n += (size_t)PAIR_CH * L.MP;                 // W2s
  n += (size_t)s.Q * PAIR_CH;                  // wqs
  if (!knn) n += (size_t)PAIR_CH * 33;         // Bs
  if (s.Q > 1) n += (size_t)s.Q * PAIR_THREADS;  // fs
  n += (size_t)4 * s.m * L.MP + 8 * s.m + 2 * L.MP + 4;   // w3s, b3s, w4s, misc
  return round_up(n * sizeof(T), 16) + 16;
}

template <typename T, int MP, bool KNN>
__global__ void __launch_bounds__(PAIR_THREADS)
pair_kernel(const PairArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Dims& s = a.s;
  const int tid = threadIdx.x;
  const int TS = a.TS, TI = PAIR_THREADS / TS;
  const int g = tid / TS, sl = tid % TS;
  const int b = blockIdx.y;
  const int i_raw = s.row0 + blockIdx.x * TI + g;
  const bool row_valid = i_raw < s.row1;
  const int i = row_valid ? i_raw : s.row0;
  const int J = KNN ? s.k : s.N;
  const int U = 4 * s.m;
  const int qd = 2 * s.F;                      // index of the raw squared distance in the Q channels
  const bool upd_feats = a.flags & EGNN_FLAG_UPDATE_FEATS;
  const bool upd_coors = a.flags & EGNN_FLAG_UPDATE_COORS;

  // ---- shared memory carve-up
  T* W2s = reinterpret_cast<T*>(smem_raw);                 // [CH][MP]
  T* wqs = W2s + PAIR_CH * MP;                             // [Q][CH]
  T* Bs = wqs + s.Q * PAIR_CH;                             // [CH][33]      (dense only)
  T* fs = Bs + (KNN ? 0 : PAIR_CH * 33);                   // [Q][128]      (Q > 1 only)
  T* w3s = fs + (s.Q > 1 ? s.Q * PAIR_THREADS : 0);        // [U][MP]
  T* b3s = w3s + U * MP;                                   // [U]
  T* w4s = b3s + U;                                        // [U]
  T* misc = w4s + U;                                       // b2[MP] | gate_w[MP] | gate_b, b4, scale

  const T* pk = a.packed;
  if (upd_coors) {
    for (int x = tid; x < U * MP; x += PAIR_THREADS) w3s[x] = pk[a.L.w3 + x];
    for (int x = tid; x < U; x += PAIR_THREADS) { b3s[x] = pk[a.L.b3 + x]; w4s[x] = pk[a.L.w4 + x]; }
  }
  for (int x = tid; x < 2 * MP + 4; x += PAIR_THREADS) misc[x] = pk[a.L.misc + x];
  // (visibility is guaranteed by the __syncthreads inside the chunk loop below)

  const T* xi = a.coors + ((size_t)b * s.N + i) * s.C;
  const bool mask_i = a.has_mask ? (a.mask[(size_t)b * s.N + i] != 0) : true;
  const T* Arow = a.P + ((size_t)b * s.N + i) * a.ldP;

  T msum[MP];
  T csum[PAIR_CMAX];
#pragma unroll
  for (int o = 0; o < MP; ++o) msum[o] = T(0);
#pragma unroll
  for (int c = 0; c < PAIR_CMAX; ++c) csum[c] = T(0);
  T cnt = T(0);

  for (int s0 = 0; s0 < J; s0 += TS) {
    const int sidx = s0 + sl;
    bool pair_valid = row_valid && sidx < J;
    int j = 0;
    bool ok = true;
    if (KNN) {
      if (pair_valid) {
        size_t o = ((size_t)b * s.N + i) * s.k + sidx;
        j = a.nbr_idx[o];
        ok = a.nbr_ok ? a.nbr_ok[o] != 0 : true;
        if (j < 0) { j = 0; pair_valid = false; }      // empty slot of a caller-supplied neighbour list
      }
    } else {
      j = pair_valid ? sidx : 0;
    }
    // ---- geometry (egnn_pytorch.py:232-233)
    T rel[PAIR_CMAX];
    T d = T(0);
    {
      const T* xj = a.coors + ((size_t)b * s.N + j) * s.C;
#pragma unroll
      for (int c = 0; c < PAIR_CMAX; ++c) {
        rel[c] = T(0);
        if (c < s.C) { rel[c] = xi[c] - xj[c]; d = sq_acc<T>(rel[c], d); }
      }
    }
    // ---- per-pair scalar channels other than d go through shared memory
    if (s.Q > 1) {
      for (int q = 0; q < s.Q; ++q) {
        T f;
        if (q < s.F) f = sin(d / T(1 << q));                     // fourier_encode_dist :34-41
        else if (q < 2 * s.F) f = cos(d / T(1 << (q - s.F)));
        else if (q == qd) f = d;
        else f = a.edges[(((size_t)b * s.N + i) * s.N + j) * s.edge_dim + (q - s.Qd)];
        fs[q * PAIR_THREADS + tid] = f;
      }
    }
    int lab = 0;
    if (a.labels) lab = a.labels[((size_t)b * s.N + i) * s.N + j];
    const T* Brow = a.P + ((size_t)b * s.N + j) * a.ldP + s.Hp;
    const T* tabrow = pk + a.L.tab + (size_t)lab * s.Hp;

    Pk2<T> accp[MP / 2];
#pragma unroll
    for (int o = 0; o < MP / 2; ++o) accp[o] = Pk2<T>::make(T(0), T(0));

    for (int c0 = 0; c0 < s.Hp; c0 += PAIR_CH) {
      const int cn = min(PAIR_CH, s.Hp - c0);      // multiple of 8
      __syncthreads();                             // previous chunk fully consumed
      for (int x = tid; x < cn * MP; x += PAIR_THREADS) W2s[x] = pk[a.L.w2t + (size_t)c0 * MP + x];
      for (int x = tid; x < s.Q * cn; x += PAIR_THREADS) {
        int q = x / cn, cc = x % cn;
        wqs[q * PAIR_CH + cc] = pk[a.L.wq + (size_t)q * s.Hp + c0 + cc];
      }
      if (!KNN) {
        // B tile, transposed: Bs[cc][jj] = B[s0 + jj][c0 + cc]
        const int cc = tid % PAIR_CH, jj0 = tid / PAIR_CH;
        for (int jj = jj0; jj < 32; jj += PAIR_THREADS / PAIR_CH) {
          T v = T(0);
          if (cc < cn && s0 + jj < s.N) v = a.P[((size_t)b * s.N + s0 + jj) * a.ldP + s.Hp + c0 + cc];
          Bs[cc * 33 + jj] = v;
        }
      }
      __syncthreads();

      for (int cc = 0; cc < cn; cc += 4) {
        Vec4<T> av, wd;
        av.load_g(Arow + c0 + cc);
        wd.load(wqs + qd * PAIR_CH + cc);
        T pre[4];
        if (KNN) {
          Vec4<T> bv;
          bv.load_g(Brow + c0 + cc);
#pragma unroll
          for (int u = 0; u < 4; ++u) pre[u] = av.v[u] + bv.v[u];
        } else {
#pragma unroll
          for (int u = 0; u < 4; ++u) pre[u] = av.v[u] + Bs[(cc + u) * 33 + sl];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) pre[u] = fma_t(wd.v[u], d, pre[u]);
        if (s.Q > 1) {
          for (int q = 0; q < s.Q; ++q) {
            if (q == qd) continue;
            const T f = fs[q * PAIR_THREADS + tid];
            Vec4<T> wv;
            wv.load(wqs + q * PAIR_CH + cc);
#pragma unroll
            for (int u = 0; u < 4; ++u) pre[u] = fma_t(wv.v[u], f, pre[u]);
          }
        }
        if (a.labels) {
          Vec4<T> tv;
          tv.load_g(tabrow + c0 + cc);
#pragma unroll
          for (int u = 0; u < 4; ++u) pre[u] += tv.v[u];
        }
        if (a.drop.thr) {                                // edge_mlp Dropout, egnn_pytorch.py:180
          const unsigned long long pkey = (((unsigned long long)b * s.N + i) * s.N + j) * s.Hp + c0 + cc;
#pragma unroll
          for (int u = 0; u < 4; ++u) pre[u] *= (T)drop_mul(a.drop, 0u, pkey + u);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const T hv = silu_acc<T>(pre[u]);             // egnn_pytorch.py:181
          const Pk2<T> hdn = Pk2<T>::make(hv, hv);
          const T* w2 = W2s + (cc + u) * MP;
#pragma unroll
          for (int v4 = 0; v4 < MP; v4 += 4) {
            Vec4<T> wv;
            wv.load(w2 + v4);
            accp[v4 / 2].fma(hdn, Pk2<T>::make(wv.v[0], wv.v[1]));
            accp[v4 / 2 + 1].fma(hdn, Pk2<T>::make(wv.v[2], wv.v[3]));
          }
        }
      }
    }
    T acc[MP];
#pragma unroll
    for (int o = 0; o < MP; o += 2) { acc[o] = accp[o / 2].lo(); acc[o + 1] = accp[o / 2].hi(); }

    if (a.pre2_out && pair_valid) {                  // kept for backward: [B,N,J][MP], J = N (dense) or k
      T* dst = a.pre2_out + (KNN ? ((size_t)b * s.N + i) * s.k + sidx : ((size_t)b * s.N + i) * s.N + j) * MP;
#pragma unroll
      for (int o = 0; o < MP; ++o) dst[o] = acc[o];
    }
    // ---- epilogue for this pair: m_ij, gate, coordinate weight, masks (egnn_pytorch.py:287-322)
    T mm[MP];
#pragma unroll
    for (int o = 0; o < MP; ++o) mm[o] = silu_acc<T>(acc[o] + misc[o]);     // pad lanes: silu(0) = 0
    if (a.flags & EGNN_FLAG_SOFT_EDGES) {
      T z = misc[2 * MP + 0];
#pragma unroll
      for (int o = 0; o < MP; ++o) z = fma_t(misc[MP + o], mm[o], z);
      const T gate = sigmoid_acc<T>(z);
#pragma unroll
      for (int o = 0; o < MP; ++o) mm[o] *= gate;
    }
    bool pm = pair_valid;
    if (a.has_mask) {
      const bool mask_j = a.mask[(size_t)b * s.N + j] != 0;
      pm = pm && mask_i && mask_j && (KNN ? ok : true);
    }
    if (upd_coors) {
      T w = misc[2 * MP + 1];
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
        if (a.drop.thr) t *= (T)drop_mul(a.drop, 1u, (((unsigned long long)b * s.N + i) * s.N + j) * U + u);    // coors_mlp Dropout, :205
        w = fma_t(w4s[u], silu_acc<T>(t), w);
      }
      if (!pm) w = T(0);                                   // :309 (and padding lanes of the tile)
      if (a.flags & EGNN_FLAG_CLAMP) w = w < -a.clamp ? -a.clamp : (w > a.clamp ? a.clamp : w);   // :313
      if (!pair_valid) w = T(0);
      T scale = T(1);
      if (a.flags & EGNN_FLAG_NORM_COORS) {                // CoorsNorm :74-77
        const T nrm = sqrt(d);
        scale = misc[2 * MP + 2] / (nrm > T(1e-8) ? nrm : T(1e-8));
      }
      w *= scale;
#pragma unroll
      for (int c = 0; c < PAIR_CMAX; ++c) csum[c] = fma_t(w, rel[c], csum[c]);
    }
    if (upd_feats && pm) {
#pragma unroll
      for (int o = 0; o < MP; ++o) msum[o] += mm[o];
      cnt += T(1);
    }
  }

  // ---- reduce over the TS lanes of the row group, then write
  for (int off = TS >> 1; off > 0; off >>= 1) {
#pragma unroll
    for (int o = 0; o < MP; ++o) msum[o] += shfl_xor_t<T>(msum[o], off);
#pragma unroll
    for (int c = 0; c < PAIR_CMAX; ++c) csum[c] += shfl_xor_t<T>(csum[c], off);
    cnt += shfl_xor_t<T>(cnt, off);
  }
  if (sl == 0 && row_valid) {
    const size_t node = (size_t)b * s.N + i;
    if (upd_feats) {
      T inv = T(1);
      if (a.flags & EGNN_FLAG_POOL_MEAN) {
        if (a.has_mask) inv = cnt > T(0) ? T(1) / cnt : T(0);     // safe_div :13-16, :327-328
        else inv = T(1) / T(J);                                    // :330
      }
#pragma unroll
      for (int o = 0; o < MP; ++o)
        if (o < s.m) a.m_out[node * a.ld_m + o] = msum[o] * inv;
    }
    if (upd_coors) {
#pragma unroll
      for (int c = 0; c < PAIR_CMAX; ++c)
        if (c < s.C) a.coors_out[node * s.C + c] = csum[c] + xi[c];   // :315
    }
  }
}

// =====================================================================================
// Dense all-pairs variant with register tiling over rows: a thread owns neighbour j and PP query rows, so every
// W2 row fetched from shared memory feeds PP pairs (the thread-per-pair kernel above is bound by the 16
// broadcast wavefronts per hidden channel that W2 costs).  One warp = PP rows x 32 neighbours,
// 4 warps per CTA; per-row sums are reduced with shuffles per j-tile and kept in shared memory.
// =====================================================================================
template <typename T>
inline size_t pair_tiled_smem_bytes(const Dims& s, const SimtPackLayout& L, int PP) {
  size_t n = 0;
  n += (size_t)PAIR_CH * L.MP;                         // W2s
  n += (size_t)s.Q * PAIR_CH;                          // wqs
  n += (size_t)PAIR_CH * 33;                           // Bs
  if (s.Q > 1) n += (size_t)PP * s.Q * PAIR_THREADS;   // fs
  n += (size_t)4 * s.m * L.MP + 8 * s.m + 2 * L.MP + 4;   // w3s, b3s, w4s, misc
  n += (size_t)4 * PP * (L.MP + PAIR_CMAX + 4);        // per-row running sums
  return round_up(n * sizeof(T), 16) + 16;
}

template <typename T, int MP, int PP>
__global__ void __launch_bounds__(PAIR_THREADS)
pair_dense_tiled_kernel(const PairArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Dims& s = a.s;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.y;
  const int U = 4 * s.m;
  const int qd = 2 * s.F;
  constexpr int RS = MP + PAIR_CMAX + 4;          // row-sum record: m[MP] | csum[CMAX] | cnt | pad
  const bool upd_feats = a.flags & EGNN_FLAG_UPDATE_FEATS;
  const bool upd_coors = a.flags & EGNN_FLAG_UPDATE_COORS;

  T* W2s = reinterpret_cast<T*>(smem_raw);
  T* wqs = W2s + PAIR_CH * MP;
  T* Bs = wqs + s.Q * PAIR_CH;
  T* fs = Bs + PAIR_CH * 33;
  T* w3s = fs + (s.Q > 1 ? PP * s.Q * PAIR_THREADS : 0);
  T* b3s = w3s + U * MP;
  T* w4s = b3s + U;
  T* misc = w4s + U;
  T* rows = misc + 2 * MP + 4;                    // [4 warps][PP][RS]

  const T* pk = a.packed;
  if (upd_coors) {
    for (int x = tid; x < U * MP; x += PAIR_THREADS) w3s[x] = pk[a.L.w3 + x];
    for (int x = tid; x < U; x += PAIR_THREADS) { b3s[x] = pk[a.L.b3 + x]; w4s[x] = pk[a.L.w4 + x]; }
  }
  for (int x = tid; x < 2 * MP + 4; x += PAIR_THREADS) misc[x] = pk[a.L.misc + x];
  for (int x = tid; x < 4 * PP * RS; x += PAIR_THREADS) rows[x] = T(0);
  __syncthreads();                                // constants visible (phase 2 never enters the chunk loop)

  int irow[PP];
  bool rvalid[PP], mask_i[PP];
  const T* Arow[PP];
#pragma unroll
  for (int p = 0; p < PP; ++p) {
    const int ir = s.row0 + (blockIdx.x * 4 + warp) * PP + p;
    rvalid[p] = ir < s.row1;
    irow[p] = rvalid[p] ? ir : s.row0;
    mask_i[p] = a.has_mask ? (a.mask[(size_t)b * s.N + irow[p]] != 0) : true;
    Arow[p] = a.P + ((size_t)b * s.N + irow[p]) * a.ldP;
  }
  T* myrows = rows + (size_t)warp * PP * RS;

  for (int s0 = 0; s0 < s.N; s0 += 32) {
    const int jraw = s0 + lane;
    const bool jv = jraw < s.N;
    const int j = jv ? jraw : 0;
    T xj[PAIR_CMAX];
    {
      const T* xjp = a.coors + ((size_t)b * s.N + j) * s.C;
#pragma unroll
      for (int c = 0; c < PAIR_CMAX; ++c) xj[c] = c < s.C ? xjp[c] : T(0);
    }
    T d[PP];
    int lab[PP];
#pragma unroll
    for (int p = 0; p < PP; ++p) {
      const T* xi = a.coors + ((size_t)b * s.N + irow[p]) * s.C;
      T dd = T(0);
#pragma unroll
      for (int c = 0; c < PAIR_CMAX; ++c)
        if (c < s.C) dd = sq_acc<T>(xi[c] - xj[c], dd);
      d[p] = dd;
      lab[p] = a.labels ? a.labels[((size_t)b * s.N + irow[p]) * s.N + j] : 0;
      if (s.Q > 1) {
        for (int q = 0; q < s.Q; ++q) {
          T f;
          if (q < s.F) f = sin(dd / T(1 << q));
          else if (q < 2 * s.F) f = cos(dd / T(1 << (q - s.F)));
          else if (q == qd) f = dd;
          else f = a.edges[(((size_t)b * s.N + irow[p]) * s.N + j) * s.edge_dim + (q - s.Qd)];
          fs[(p * s.Q + q) * PAIR_THREADS + tid] = f;
        }
      }
    }

    Pk2<T> accp[PP][MP / 2];
#pragma unroll
    for (int p = 0; p < PP; ++p)
#pragma unroll
      for (int o = 0; o < MP / 2; ++o) accp[p][o] = Pk2<T>::make(T(0), T(0));

    int c_begin = 0, c_end = s.Hp;
    if (a.phase == 1) {
      const int per = ceil_div(ceil_div(s.Hp, PAIR_CH), a.hsplit) * PAIR_CH;
      c_begin = blockIdx.z * per;
      c_end = min(s.Hp, c_begin + per);
    } else if (a.phase == 2) {
      c_end = 0;
    }
    for (int c0 = c_begin; c0 < c_end; c0 += PAIR_CH) {
      const int cn = min(PAIR_CH, s.Hp - c0);
      __syncthreads();
      for (int x = tid; x < cn * MP; x += PAIR_THREADS) W2s[x] = pk[a.L.w2t + (size_t)c0 * MP + x];
      for (int x = tid; x < s.Q * cn; x += PAIR_THREADS) {
        int q = x / cn, cc = x % cn;
        wqs[q * PAIR_CH + cc] = pk[a.L.wq + (size_t)q * s.Hp + c0 + cc];
      }
      {
        const int cc = tid % PAIR_CH, jj0 = tid / PAIR_CH;
        for (int jj = jj0; jj < 32; jj += PAIR_THREADS / PAIR_CH) {
          T v = T(0);
          if (cc < cn && s0 + jj < s.N) v = a.P[((size_t)b * s.N + s0 + jj) * a.ldP + s.Hp + c0 + cc];
          Bs[cc * 33 + jj] = v;
        }
      }
      __syncthreads();

      for (int cc = 0; cc < cn; cc += 4) {
        Vec4<T> wd;
        wd.load(wqs + qd * PAIR_CH + cc);
        T bv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) bv[u] = Bs[(cc + u) * 33 + lane];
        T pre[PP][4];
#pragma unroll
        for (int p = 0; p < PP; ++p) {
          Vec4<T> av;
          av.load_g(Arow[p] + c0 + cc);
#pragma unroll
          for (int u = 0; u < 4; ++u) pre[p][u] = fma_t(wd.v[u], d[p], av.v[u] + bv[u]);
          if (a.labels) {
            Vec4<T> tv;
            tv.load_g(pk + a.L.tab + (size_t)lab[p] * s.Hp + c0 + cc);
#pragma unroll
            for (int u = 0; u < 4; ++u) pre[p][u] += tv.v[u];
          }
        }
        if (s.Q > 1) {
          for (int q = 0; q < s.Q; ++q) {
            if (q == qd) continue;
            Vec4<T> wv;
            wv.load(wqs + q * PAIR_CH + cc);
#pragma unroll
            for (int p = 0; p < PP; ++p) {
              const T f = fs[(p * s.Q + q) * PAIR_THREADS + tid];
#pragma unroll
              for (int u = 0; u < 4; ++u) pre[p][u] = fma_t(wv.v[u], f, pre[p][u]);
            }
          }
        }
        if (a.drop.thr) {                                // edge_mlp Dropout, egnn_pytorch.py:180
#pragma unroll
          for (int p = 0; p < PP; ++p) {
            const unsigned long long pkey = (((unsigned long long)b * s.N + irow[p]) * s.N + j) * s.Hp + c0 + cc;
#pragma unroll
            for (int u = 0; u < 4; ++u) pre[p][u] *= (T)drop_mul(a.drop, 0u, pkey + u);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const T* w2 = W2s + (cc + u) * MP;
          Pk2<T> hdn[PP];
#pragma unroll
          for (int p = 0; p < PP; ++p) {
            const T hv = silu_acc<T>(pre[p][u]);
            hdn[p] = Pk2<T>::make(hv, hv);
          }
#pragma unroll
          for (int v4 = 0; v4 < MP; v4 += 4) {
            Vec4<T> wv;
            wv.load(w2 + v4);
            const Pk2<T> w01 = Pk2<T>::make(wv.v[0], wv.v[1]), w23 = Pk2<T>::make(wv.v[2], wv.v[3]);
#pragma unroll
            for (int p = 0; p < PP; ++p) {
              accp[p][v4 / 2].fma(hdn[p], w01);
              accp[p][v4 / 2 + 1].fma(hdn[p], w23);
            }
          }
        }
      }
    }
    T acc[PP][MP];
#pragma unroll
    for (int p = 0; p < PP; ++p)
#pragma unroll
      for (int o = 0; o < MP; o += 2) { acc[p][o] = accp[p][o / 2].lo(); acc[p][o + 1] = accp[p][o / 2].hi(); }

    if (a.phase != 0) {
      // split hidden axis: partial sums go through global memory, summed in split order (deterministic)
#pragma unroll
      for (int p = 0; p < PP; ++p) {
        if (!(rvalid[p] && jv)) continue;
        const size_t pair = ((size_t)b * s.N + irow[p]) * s.N + j;
        const size_t stride = (size_t)s.B * s.N * s.N * MP;
        if (a.phase == 1) {
#pragma unroll
          for (int o = 0; o < MP; ++o) a.hpart[blockIdx.z * stride + pair * MP + o] = acc[p][o];
        } else {
          for (int z = 0; z < a.hsplit; ++z)
#pragma unroll
            for (int o = 0; o < MP; ++o) acc[p][o] += a.hpart[z * stride + pair * MP + o];
        }
      }
      if (a.phase == 1) continue;
    }
    if (a.pre2_out) {
#pragma unroll
      for (int p = 0; p < PP; ++p) {
        if (!(rvalid[p] && jv)) continue;
        T* dst = a.pre2_out + (((size_t)b * s.N + irow[p]) * s.N + j) * MP;
#pragma unroll
        for (int o = 0; o < MP; ++o) dst[o] = acc[p][o];
      }
    }
    // ---- epilogue of this j-tile for the PP rows
    const bool mask_j = a.has_mask ? (a.mask[(size_t)b * s.N + j] != 0) : true;
#pragma unroll
    for (int p = 0; p < PP; ++p) {
      T mm[MP];
#pragma unroll
      for (int o = 0; o < MP; ++o) mm[o] = silu_acc<T>(acc[p][o] + misc[o]);
      if (a.flags & EGNN_FLAG_SOFT_EDGES) {
        T z = misc[2 * MP + 0];
#pragma unroll
        for (int o = 0; o < MP; ++o) z = fma_t(misc[MP + o], mm[o], z);
        const T gate = sigmoid_acc<T>(z);
#pragma unroll
        for (int o = 0; o < MP; ++o) mm[o] *= gate;
      }
      const bool pair_valid = rvalid[p] && jv;
      const bool pm = pair_valid && (a.has_mask ? (mask_i[p] && mask_j) : true);
      T rec[RS];
#pragma unroll
      for (int x = 0; x < RS; ++x) rec[x] = T(0);
      if (upd_coors) {
        T w = misc[2 * MP + 1];
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
          if (a.drop.thr) t *= (T)drop_mul(a.drop, 1u, (((unsigned long long)b * s.N + irow[p]) * s.N + j) * U + u);   // :205
          w = fma_t(w4s[u], silu_acc<T>(t), w);
        }
        if (!pm) w = T(0);
        if (a.flags & EGNN_FLAG_CLAMP) w = w < -a.clamp ? -a.clamp : (w > a.clamp ? a.clamp : w);
        if (!pair_valid) w = T(0);
        if (a.flags & EGNN_FLAG_NORM_COORS) {
          const T nrm = sqrt(d[p]);
          w *= misc[2 * MP + 2] / (nrm > T(1e-8) ? nrm : T(1e-8));
        }
        const T* xi = a.coors + ((size_t)b * s.N + irow[p]) * s.C;
#pragma unroll
        for (int c = 0; c < PAIR_CMAX; ++c)
          if (c < s.C) rec[MP + c] = w * (xi[c] - xj[c]);
      }
      if (upd_feats && pm) {
#pragma unroll
        for (int o = 0; o < MP; ++o) rec[o] = mm[o];
        rec[MP + PAIR_CMAX] = T(1);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int x = 0; x < MP + PAIR_CMAX + 1; ++x) rec[x] += shfl_xor_t<T>(rec[x], off);
      if (lane == 0) {
#pragma unroll
        for (int x = 0; x < MP + PAIR_CMAX + 1; ++x) myrows[p * RS + x] += rec[x];
      }
    }
  }

  __syncwarp();
  if (a.phase != 1 && lane < PP && rvalid[0]) {
    // lane p writes row p (rvalid is monotone in p)
    int p = lane;
    const int ir = s.row0 + (blockIdx.x * 4 + warp) * PP + p;
    if (ir < s.row1) {
      const size_t node = (size_t)b * s.N + ir;
      const T* rec = myrows + p * RS;
      if (upd_feats) {
        T inv = T(1);
        if (a.flags & EGNN_FLAG_POOL_MEAN) {
          const T cnt = rec[MP + PAIR_CMAX];
          if (a.has_mask) inv = cnt > T(0) ? T(1) / cnt : T(0);
          else inv = T(1) / T(s.N);
        }
        for (int o = 0; o < s.m; ++o) a.m_out[node * a.ld_m + o] = rec[o] * inv;
      }
      if (upd_coors) {
        const T* xi = a.coors + node * s.C;
        for (int c = 0; c < s.C; ++c) a.coors_out[node * s.C + c] = rec[MP + c] + xi[c];
      }
    }
  }
}

}  // namespace egnn

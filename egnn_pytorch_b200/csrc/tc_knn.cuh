// The fused edge step on tensor cores for neighbour lists (any k, bf16 operands).
//
// Reference semantics: the use_nearest branch of EGNN.forward -- gathers of rel_coors / rel_dist / edges / feats
// along the selected neighbours (egnn_pytorch.py:262-266, :275), edge MLP (:287), gate (:289-290), neighbour
// mask incl. valid_radius (:292-300), coors MLP / clamp / CoorsNorm (:302-315), pooling (:319-333).  The
// neighbour lists come from egnn_knn_select (knn_select.cu).
//
// Same machinery as tc_pair.cuh (hidden values produced in fp32 registers and packed to bf16 directly in the
// mma.sync A-fragment layout, m16n8k16 MMAs against the W2 slab in shared memory, accumulators in registers).
// What differs:
//   * one WARP owns one query row i and its 32 neighbour slots (slot >= k is padding), so the reduction over j is a
//     single warp shuffle tree;
//   * k > 32 (WIDE): the warp runs the row's slots in groups of 32, one after another -- per group it re-gathers the
//     neighbour indices, pair vectors, edge channels / scalar tile and B' rows, and reuses everything staged per CTA
//     (A' rows, W2 slabs, Wq / We tables, epilogue constants) and per row (box or cell); each group's record is
//     shuffle-reduced and summed one channel per lane in shared memory, so no register lives across the groups;
//   * the B' row of every pair is gathered from L2 (8-byte pieces, contiguous across the 4 lanes that share a
//     pair) and used once: each 64-channel round re-fills its B' registers for the next chunk right after use;
//   * up to 4 continuous edge channels per pair are folded in on the CUDA cores (We from shared memory);
//   * MODE 2 is the generic instantiation: any number (<= TP_QMAX) of per-pair scalar channels -- squared distance,
//     fourier features (egnn_pytorch.py:34-41), continuous edge channels, one-hot adjacency-degree labels (the folded
//     `adj_emb` of EGNN_Network, :430-432) -- kept per slot in a small per-warp shared-memory tile, and any coordinate
//     dimension C <= 8.  BASELINE config 5 (only_sparse_neighbors + num_adj_degrees) runs here.
#pragma once

#include <cuda_bf16.h>
#include "common.cuh"
#include "tc_common.cuh"
#include "tc_pair.cuh"     // TP_EPI_FLOATS and the epilogue constant layout

namespace egnn {

constexpr int TK_ROWS = 16;        // query rows per CTA (one per warp): 16, or 8 when two CTAs then fit on an SM
constexpr int TK_KC = 64;
constexpr int TK_ACC_LD = 18;      // floats per slot row of the per-warp accumulator transpose tile
constexpr int TK_QE = 4;           // edge channels folded per pair (edge_dim <= 4, zero padded)

constexpr int TK_LEAN = 0, TK_EDGES = 1, TK_GEN = 2;

struct TcKnnArgs {
  int B, N, Hp, ldn, dim, k, edge_dim;
  int C, Q, F, num_labels;         // generic instantiation: Q = 1 + 2F + edge_dim + num_labels channels, C coordinates
  int row0, row1;                  // i-rows [row0, row1) of every graph are evaluated
  uint32_t flags; int has_mask; float clamp;
  const float* Atab;               // [M][Hp]  0.5 (h W1_i^T + b1)
  const __nv_bfloat16* Btab;       // [M][Hp]  0.5 h W1_j^T
  const float* wdh;                // [Hp]     0.5 W1[:, 2dim]                        (= row 0 of the packed Wq table)
  const float* weh;                // [TK_QE][Hp]  0.5 W1[:, 2dim+1+q]  (zero rows beyond edge_dim; rows 1..4 of Wq)
  const uint8_t* labels;           // [B][N][N] | null  (generic instantiation)
  const __nv_bfloat16* w2p;        // W2 in core-matrix order
  const float* epi;
  const float* coors;              // [B][N][3]
  const __nv_bfloat16* edges;      // [B][N][N][edge_dim], [B][N][k][edge_dim] under EGNN_FLAG_EDGES_PER_SLOT, | null
  const uint8_t* mask;             // [B][N] | null
  const int32_t* nbr_idx;          // [B][N][k]
  const uint8_t* nbr_ok;           // [B][N][k]
  __nv_bfloat16* m_out;            // node_in + dim (stride ldn) | null
  float* coors_out;                // [B][N][3] | null
  const float* box;                // [B][C] periodic box lengths (PBC_BOX) or [B][C][C] cell (PBC_CELL)
};

// channels of the Wq table staged in shared memory: 1 (lean), 1 + TK_QE (edges), Q (generic)
inline int tc_knn_wq_rows(int mode, int Q) { return mode == TK_LEAN ? 1 : mode == TK_EDGES ? 1 + TK_QE : Q; }

inline size_t tc_knn_smem_bytes(int Hp, int mode, int Q = 1, int rows = TK_ROWS) {
  size_t n = 0;
  n += (size_t)Hp * 32;                       // W2 slabs
  n += (size_t)rows * Hp * 4;                 // A rows (fp32)
  n += (size_t)tc_knn_wq_rows(mode, Q) * Hp * 4;   // wd | We | generic Wq
  n += (size_t)TP_EPI_FLOATS * 4;             // epilogue constants
  n += mode == TK_GEN ? (size_t)rows * Q * 32 * 4 : 0;   // per-warp scalar tile [Q][32 slots]
  n += (size_t)rows * 32 * TK_ACC_LD * 4;     // per-warp accumulator transpose tile [32 slots][TK_ACC_LD]
  n += 64 + 8;                                // mbarrier
  return n + 128;
}

// Rows per CTA: a CTA runs its prologue (staging W2 / A' / channel weights, the dependent gathers of
// neighbour indices, coordinates and edge channels), 17-odd chunks and the coors-MLP epilogue back to back, so with one
// CTA per SM the MUFU pipe idles through every prologue and epilogue (c4: 52 us per CTA for 19 us of MUFU work).  With
// ROWS = 8 (256 threads, half the A' rows) two CTAs are resident and cover each other's phases; the
// host takes ROWS = 8 whenever two CTAs fit in shared memory (rows_per_cta below).
inline int tc_knn_rows_per_cta(int Hp, int mode, int Q) { return 2 * (tc_knn_smem_bytes(Hp, mode, Q, 8) + 1024) <= 227 * 1024 ? 8 : 16; }

// PBC: rel is the minimum image under a.box (PBC_BOX) or wrapped by the cell a.box (PBC_CELL); the distance and the
// coordinate sum both follow from it
template <int MODE, int ROWS, int PBC = PBC_NONE, bool WIDE = false>
__global__ void __launch_bounds__(ROWS * 32, ROWS == 8 ? 2 : 1) tc_knn_kernel(const TcKnnArgs a) {
  constexpr int TK_THREADS = ROWS * 32;
  constexpr bool EDGES = MODE == TK_EDGES, GEN = MODE == TK_GEN;
  constexpr int NX = GEN ? TP_CMAX : 3;                                       // coordinate registers
  constexpr int PW = GEN ? 16 + TP_CMAX + 1 : 20;                             // reduced record: 16 m | coords | count
  static_assert(PW <= 32 && TK_ACC_LD > 16, "WIDE keeps one record channel per lane in a padding column of accs");
  extern __shared__ __align__(128) unsigned char sm[];
  const int Hp = a.Hp, N = a.N, K = a.k;
  const int C = GEN ? a.C : 3, Q = GEN ? a.Q : 1;
  unsigned char* w2s = sm;
  float* As = reinterpret_cast<float*>(w2s + (size_t)Hp * 32);                // [16][Hp]
  float* wds = As + (size_t)ROWS * Hp;                                     // [Hp]  (generic: Wq [Q][Hp])
  float* wes = wds + Hp;                                                      // [QE][Hp] (EDGES only)
  float* epi = wds + (size_t)(GEN ? Q : EDGES ? 1 + TK_QE : 1) * Hp;
  float* stile = epi + TP_EPI_FLOATS;                                         // [16 warps][Q][32] (GEN only)
  float* accs = stile + (GEN ? ROWS * Q * 32 : 0);                            // [16 warps][32][TK_ACC_LD]
  uint64_t* ldbar = reinterpret_cast<uint64_t*>(accs + ROWS * 32 * TK_ACC_LD);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.y, i0 = a.row0 + blockIdx.x * ROWS;
  const int rows_valid = min(ROWS, a.row1 - i0);
  const int nchunks = (Hp + TK_KC - 1) / TK_KC;
  const int nsl_last = (Hp - (nchunks - 1) * TK_KC) / 16;        // valid K slabs of the last chunk (Hp is a multiple of 16)
  const bool upd_feats = a.flags & EGNN_FLAG_UPDATE_FEATS, upd_coors = a.flags & EGNN_FLAG_UPDATE_COORS;

  if (tid == 0) {
    tc::mbar_init(ldbar, 1);
    tc::mbar_fence_init();
  }
  for (int x = tid; x < TP_EPI_FLOATS; x += TK_THREADS) epi[x] = a.epi[x];
  for (int x = tid + rows_valid * Hp; x < ROWS * Hp; x += TK_THREADS) As[x] = 0.f;
  __syncthreads();

  if (tid == 0) {
    const uint32_t w2_bytes = (uint32_t)Hp * 32, as_bytes = (uint32_t)rows_valid * Hp * 4;
    const uint32_t wd_bytes = (uint32_t)(GEN ? Q : 1) * Hp * 4;              // generic: the whole Wq table (rows are contiguous)
    const uint32_t we_bytes = EDGES ? (uint32_t)TK_QE * Hp * 4 : 0u;
    tc::mbar_arrive_expect_tx(ldbar, w2_bytes + as_bytes + wd_bytes + we_bytes);
    auto bulk = [&](uint32_t dst, const unsigned char* src, uint32_t bytes) {
      for (uint32_t o = 0; o < bytes; o += 16384) tc::tma_bulk_g2s(dst + o, src + o, min(16384u, bytes - o), ldbar);
    };
    bulk(tc::smem_u32(w2s), reinterpret_cast<const unsigned char*>(a.w2p), w2_bytes);
    bulk(tc::smem_u32(As), reinterpret_cast<const unsigned char*>(a.Atab + ((size_t)b * N + i0) * Hp), as_bytes);
    bulk(tc::smem_u32(wds), reinterpret_cast<const unsigned char*>(a.wdh), wd_bytes);
    if (EDGES) bulk(tc::smem_u32(wes), reinterpret_cast<const unsigned char*>(a.weh), we_bytes);
  }

  const int lr = lane >> 2, lq = lane & 3;

  // ---- this warp's query row
  const bool iv = warp < rows_valid;
  const int i = i0 + (iv ? warp : 0);
  const size_t nodei = (size_t)b * N + i;
  float xi[NX];
#pragma unroll
  for (int c = 0; c < NX; ++c) xi[c] = (!GEN || c < C) ? a.coors[nodei * C + c] : 0.f;
  const bool mask_i = iv && (a.has_mask ? a.mask[nodei] != 0 : true);

  float boxL = 0.f, boxinv = 0.f;                      // PBC: lane c holds axis c of this graph's box, once per row
  float cv = 0.f;                                      // PBC_CELL: lane t < 9 holds value t of this graph's staged cell
  int s0 = 0;                                          // slot groups [s0, s0 + 32): the whole row unless WIDE
  do {
    if (WIDE && s0 > 0) __syncwarp();                    // the previous group's reads of myS / myacc are done
    const int slot = s0 + lane;
    // ---- pair mapping: lane = neighbour slot s0 + lane
    bool sv = iv && slot < K;
    int j = i;
    bool okj = true;
    if (sv) {
      j = a.nbr_idx[nodei * K + slot];
      okj = a.nbr_ok ? a.nbr_ok[nodei * K + slot] != 0 : true;
      if (j < 0) { j = i; sv = false; }                 // empty slot of a caller-supplied neighbour list
    }
    const size_t nodej = (size_t)b * N + j;
    float rel[NX];
    float dmine = 0.f;
    if constexpr (PBC == PBC_CELL) {                     // loaded once per row, broadcast per group (one live register)
      if (s0 == 0) cv = cell_staged<float>(a.box, b, C, lane < CELL_STAGED ? lane : 0);
      float pc[CELL_STAGED];
#pragma unroll
      for (int t = 0; t < CELL_STAGED; ++t) pc[t] = __shfl_sync(0xffffffffu, cv, t);
#pragma unroll
      for (int c = 0; c < NX; ++c) rel[c] = (!GEN || c < C) ? xi[c] - a.coors[nodej * C + c] : 0.f;
      cell_wrap<float>(rel[0], rel[1], rel[2], pc);
#pragma unroll
      for (int c = 0; c < NX; ++c) dmine = fmaf(rel[c], rel[c], dmine);
    } else {
      if constexpr (PBC) if (s0 == 0) box_axis<float>(a.box, b, C, lane < NX ? lane : NX, boxL, boxinv);
#pragma unroll
      for (int c = 0; c < NX; ++c) {
        rel[c] = (!GEN || c < C) ? xi[c] - a.coors[nodej * C + c] : 0.f;
        if constexpr (PBC)
          rel[c] = min_image<float>(rel[c], __shfl_sync(0xffffffffu, boxL, c), __shfl_sync(0xffffffffu, boxinv, c));
        dmine = fmaf(rel[c], rel[c], dmine);
      }
    }
    float* myS = stile + (size_t)warp * Q * 32;          // generic: this warp's per-slot scalar channels
    if (GEN) {
      myS[lane] = dmine;
      int q = 1;
      for (int f = 0; f < a.F; ++f) {                                                               // :34-41
        const float sc = dmine * exp2f(-(float)f);
        myS[(q + f) * 32 + lane] = sinf(sc);
        myS[(q + a.F + f) * 32 + lane] = cosf(sc);
      }
      q += 2 * a.F;
      const size_t pij = ((size_t)b * N + i) * N + j;
      const __nv_bfloat16* erow = edge_row(a.edges, a.flags & EGNN_FLAG_EDGES_PER_SLOT, nodei, slot, j, N, K, a.edge_dim);
      for (int e = 0; e < a.edge_dim; ++e) myS[(q + e) * 32 + lane] = __bfloat162float(erow[e]);
      q += a.edge_dim;
      if (a.num_labels > 0) {
        const int lab = a.labels[pij];
        for (int l = 0; l < a.num_labels; ++l) myS[(q + l) * 32 + lane] = (l == lab) ? 1.f : 0.f;
      }
      __syncwarp();
    }
    // ---- fragment mapping: rows (slots) lr + 8*rho of this warp; fetch their j, d, edges by shuffle / gather
    int jf[4];
    float dr[4];
    float ef[4][TK_QE];
#pragma unroll
    for (int rho = 0; rho < 4; ++rho) {
      jf[rho] = __shfl_sync(0xffffffffu, j, lr + 8 * rho);
      dr[rho] = __shfl_sync(0xffffffffu, dmine, lr + 8 * rho);
#pragma unroll
      for (int q = 0; q < TK_QE; ++q) ef[rho][q] = 0.f;
      if (EDGES) {      // per-slot edges: the group's 32 slots are one contiguous run of 32 * edge_dim values from slot s0
        const __nv_bfloat16* ep = edge_row(a.edges, a.flags & EGNN_FLAG_EDGES_PER_SLOT, nodei, s0 + lr + 8 * rho, jf[rho], N, K, a.edge_dim);
#pragma unroll
        for (int q = 0; q < TK_QE; ++q) if (q < a.edge_dim) ef[rho][q] = __bfloat162float(ep[q]);
      }
    }
    const uint2* Bp[4];
#pragma unroll
    for (int rho = 0; rho < 4; ++rho)
      Bp[rho] = reinterpret_cast<const uint2*>(a.Btab + ((size_t)b * N + jf[rho]) * Hp + 4 * lq);

    tc::mbar_wait(ldbar, 0);
    uint2 Bc[4][4];
    {
      const int nsl0 = nchunks == 1 ? nsl_last : 4;
#pragma unroll
      for (int rho = 0; rho < 4; ++rho)
#pragma unroll
        for (int sl = 0; sl < 4; ++sl) Bc[rho][sl] = sl < nsl0 ? __ldg(Bp[rho] + sl * 4) : make_uint2(0u, 0u);
    }

    float acc[2][2][4];                                  // m_pre of slots [16 half, +16) x channels [8 nt, +8): mma.sync D fragments
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[h][nt][e] = 0.f;

    const float* Arow = As + (size_t)warp * Hp + lq * 4;
    // chunks with all 4 K slabs run with NSLC = 4 (the slab tests fold at compile time); only the last chunk of a hidden
    // width that is not a multiple of 64 takes the predicated instantiation (NSLC = 0)
    auto chunk = [&](const int c, auto nslc) {
      constexpr int NSLC = decltype(nslc)::value;
      const bool more = NSLC != 0 && c + 1 < nchunks;
      const int nsl = NSLC ? NSLC : nsl_last, nsl_next = c + 2 == nchunks ? nsl_last : 4;
      // Slab-major: the broadcast operands of a slab (A', w_d, edge-channel weights; 16 bytes per lane each, and every
      // LDS.128 costs four L1 wavefronts whatever the overlap between lanes) are fetched ONCE and used for all four slots of
      // the thread -- the kernel is bound by L1 wavefronts (ncu: 85 % of peak, 70 % of them these loads), not by the MUFU
      // pipe.  Every (half, slab) fragment is multiplied as soon as it is packed.
#pragma unroll
      for (int sl = 0; sl < 4; ++sl) {
        if (NSLC == 0 && sl >= nsl) continue;                 // tail chunk: slabs beyond H are neither computed nor multiplied
        const float4 av = *reinterpret_cast<const float4*>(Arow + c * TK_KC + sl * 16);
        float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!GEN) wv = *reinterpret_cast<const float4*>(wds + c * TK_KC + sl * 16 + lq * 4);
        float zg[GEN ? 4 : 1][4];                              // generic: A' + sum_q Wq[q] s_q for the four slots
        if (GEN) {
#pragma unroll
          for (int rho = 0; rho < 4; ++rho) { zg[GEN ? rho : 0][0] = av.x; zg[GEN ? rho : 0][1] = av.y; zg[GEN ? rho : 0][2] = av.z; zg[GEN ? rho : 0][3] = av.w; }
#pragma unroll 1
          for (int q = 0; q < Q; ++q) {
            const float4 wq4 = *reinterpret_cast<const float4*>(wds + (size_t)q * Hp + c * TK_KC + sl * 16 + lq * 4);
#pragma unroll
            for (int rho = 0; rho < 4; ++rho) {
              const float sq = myS[q * 32 + lr + 8 * rho];
              float (&zz)[4] = zg[GEN ? rho : 0];
              zz[0] = fmaf(wq4.x, sq, zz[0]); zz[1] = fmaf(wq4.y, sq, zz[1]);
              zz[2] = fmaf(wq4.z, sq, zz[2]); zz[3] = fmaf(wq4.w, sq, zz[3]);
            }
          }
        }
        float4 we[TK_QE];
        if (EDGES) {
#pragma unroll
          for (int q = 0; q < TK_QE; ++q) we[q] = *reinterpret_cast<const float4*>(wes + (size_t)q * Hp + c * TK_KC + sl * 16 + lq * 4);
        }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          uint32_t h4[4];
#pragma unroll
          for (int r2 = 0; r2 < 2; ++r2) {
            const int rho = half * 2 + r2;
            const uint2 bb = Bc[rho][sl];
            const float d = dr[rho];
            // channel pairs (tc::ffma2: two FFMAs) for w_d d + A', the edge channels and y + y tanh y
            float2 z01, z23;
            if (GEN) {
              z01 = make_float2(zg[GEN ? rho : 0][0], zg[GEN ? rho : 0][1]); z23 = make_float2(zg[GEN ? rho : 0][2], zg[GEN ? rho : 0][3]);
            } else {
              const float2 dd = make_float2(d, d);
              z01 = tc::ffma2(make_float2(wv.x, wv.y), dd, make_float2(av.x, av.y));
              z23 = tc::ffma2(make_float2(wv.z, wv.w), dd, make_float2(av.z, av.w));
            }
            if (EDGES) {
#pragma unroll
              for (int q = 0; q < TK_QE; ++q) {
                const float2 ee = make_float2(ef[rho][q], ef[rho][q]);
                z01 = tc::ffma2(make_float2(we[q].x, we[q].y), ee, z01);
                z23 = tc::ffma2(make_float2(we[q].z, we[q].w), ee, z23);
              }
            }
            const float2 y01 = make_float2(tc::add_bf16_lo(bb.x, z01.x), tc::add_bf16_hi(bb.x, z01.y));
            const float2 y23 = make_float2(tc::add_bf16_lo(bb.y, z23.x), tc::add_bf16_hi(bb.y, z23.y));
            const float2 h01 = tc::ffma2(y01, make_float2(tc::tanh_fast(y01.x), tc::tanh_fast(y01.y)), y01);
            const float2 h23 = tc::ffma2(y23, make_float2(tc::tanh_fast(y23.x), tc::tanh_fast(y23.y)), y23);
            h4[r2 * 2 + 0] = tc::pack_bf16x2(h01.x, h01.y);
            h4[r2 * 2 + 1] = tc::pack_bf16x2(h23.x, h23.y);
            if (more && sl < nsl_next) Bc[rho][sl] = __ldg(Bp[rho] + (c + 1) * 16 + sl * 4);
          }
          // A fragment of slab sl: registers {0,1} -> slot lr (+16), {2,3} -> slot lr + 8 (+24)
          tc::mma_w2_slab(acc[half], h4, w2s, c * 4 + sl, lr, lq);
        }
      }
    };
    {
      const int nfull = nsl_last == 4 ? nchunks : nchunks - 1;
#pragma unroll 1
      for (int c = 0; c < nfull; ++c) chunk(c, tc::IntC<4>{});
      if (nfull < nchunks) chunk(nchunks - 1, tc::IntC<0>{});
    }

    // ---- epilogue (pair mapping): one warp = one query row, shuffle tree over its 32 slots
    {
      const float* W3 = epi; const float* b3 = epi + 1024; const float* w4 = b3 + 64;
      const float* b2 = w4 + 64; const float* gw = b2 + 16; const float* sc = gw + 16;
      // accumulator fragments -> one slot row per lane, through this warp's transpose tile
      float* myacc = accs + (size_t)warp * 32 * TK_ACC_LD;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int r2 = 0; r2 < 2; ++r2)
            *reinterpret_cast<float2*>(myacc + (16 * h + 8 * r2 + lr) * TK_ACC_LD + 8 * nt + 2 * lq) =
                make_float2(acc[h][nt][2 * r2], acc[h][nt][2 * r2 + 1]);
      __syncwarp();
      float m[16];
#pragma unroll
      for (int o = 0; o < 16; ++o) m[o] = tc::silu_half_arg(0.5f * (myacc[lane * TK_ACC_LD + o] + b2[o]));
      if (a.flags & EGNN_FLAG_SOFT_EDGES) {
        float z = sc[0];
#pragma unroll
        for (int o = 0; o < 16; ++o) z = fmaf(gw[o], m[o], z);
        const float gate = 0.5f + 0.5f * tc::tanh_fast(0.5f * z);
#pragma unroll
        for (int o = 0; o < 16; ++o) m[o] *= gate;
      }
      bool pm = sv;
      if (a.has_mask) pm = pm && mask_i && (a.mask[nodej] != 0) && okj;      // :296-297 (nbhd_mask only with a mask)
      float w = 0.f;
      if (upd_coors) {
        w = sc[1];
#pragma unroll 4
        for (int u = 0; u < 64; ++u) {
          const float4* w3 = reinterpret_cast<const float4*>(W3 + u * 16);
          float tt = b3[u];
#pragma unroll
          for (int o4 = 0; o4 < 4; ++o4) {
            const float4 ww = w3[o4];
            tt = fmaf(ww.x, m[o4 * 4], tt); tt = fmaf(ww.y, m[o4 * 4 + 1], tt);
            tt = fmaf(ww.z, m[o4 * 4 + 2], tt); tt = fmaf(ww.w, m[o4 * 4 + 3], tt);
          }
          w = fmaf(w4[u], tc::silu_half_arg(0.5f * tt), w);
        }
        if (!pm) w = 0.f;
        if (a.flags & EGNN_FLAG_CLAMP) w = fminf(fmaxf(w, -a.clamp), a.clamp);
        if (!sv) w = 0.f;                                                  // padding slots carry nothing, clamp or not
        if (a.flags & EGNN_FLAG_NORM_COORS) w *= sc[2] / fmaxf(sqrtf(dmine), 1e-8f);
      }
      float v[PW];
#pragma unroll
      for (int c = 0; c < NX; ++c) v[16 + c] = w * rel[c];
      v[PW - 1] = pm ? 1.f : 0.f;
#pragma unroll
      for (int o = 0; o < 16; ++o) v[o] = pm ? m[o] : 0.f;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int o = 0; o < PW; ++o) v[o] += __shfl_xor_sync(0xffffffffu, v[o], off);
      if constexpr (WIDE) {      // channel `lane` of the record, summed over the groups in the padding column of the lane's
        float mine = 0.f;        // transpose row (the transposes write columns 0..15 only): no register across the chunks
#pragma unroll
        for (int o = 0; o < PW; ++o) if (o == lane) mine = v[o];
        float& run = myacc[lane * TK_ACC_LD + 16];
        run = s0 == 0 ? mine : run + mine;
      } else if (iv) {
        if (upd_feats && lane < 16) {
          float inv = 1.f;
          if (a.flags & EGNN_FLAG_POOL_MEAN) inv = a.has_mask ? (v[PW - 1] > 0.f ? 1.f / v[PW - 1] : 0.f) : 1.f / (float)K;
          float mine = 0.f;
#pragma unroll
          for (int o = 0; o < 16; ++o) if (o == lane) mine = v[o];
          a.m_out[nodei * a.ldn + lane] = __float2bfloat16(mine * inv);
        }
        if (upd_coors && lane == 0) {
#pragma unroll
          for (int c = 0; c < NX; ++c)
            if (!GEN || c < C) a.coors_out[nodei * C + c] = xi[c] + v[16 + c];
        }
      }
    }
  } while (WIDE && (s0 += 32) < K);
  if constexpr (WIDE) {      // lane o < 16: m channel o | lane 16 + c: coordinate c | lane PW - 1: valid pairs
    const float run = accs[((size_t)warp * 32 + lane) * TK_ACC_LD + 16];
    const float cnt = __shfl_sync(0xffffffffu, run, PW - 1);
    if (iv) {
      if (upd_feats && lane < 16) {
        float inv = 1.f;
        if (a.flags & EGNN_FLAG_POOL_MEAN) inv = a.has_mask ? (cnt > 0.f ? 1.f / cnt : 0.f) : 1.f / (float)K;
        a.m_out[nodei * a.ldn + lane] = __float2bfloat16(run * inv);
      }
      const int c = lane - 16;
      if (upd_coors && c >= 0 && c < C) {
        float x = 0.f;
#pragma unroll
        for (int t = 0; t < NX; ++t) if (t == c) x = xi[t];
        a.coors_out[nodei * C + c] = x + run;
      }
    }
  }
}

}  // namespace egnn

// The fused edge step on the tensor cores (dense all-pairs, bf16 operands, fp32 accumulation).
//
// Reference semantics: egnn_pytorch.py:232-233 (x_i - x_j, squared distance), :270-285 (fourier features, edge
// input [h_i | h_j | d | e_ij]), :287 (edge MLP), :289-290 (gate), :292-333 (masks, coors MLP, clamp, both sums
// over j); EGNN_Network's adjacency-degree embedding (:430-432) enters as one-hot per-pair channels.
//
// Per pair (i, j) the split form needs  hidden[c] = SiLU(A_i[c] + B_j[c] + sum_q s_q(i,j) Wq[q][c]), c < H, and
// m_pre = hidden . W2^T  (H -> 16).  s_0 is the squared distance; the generic instantiation (GEN) adds fourier
// features, continuous edge channels and one-hot degree labels as further per-pair scalar channels, and
// handles any coordinate dimension C <= 8.
//
// PERSISTENT kernel: one CTA per SM walks "row groups" (TI = 4 query rows i of one graph) with a static stride.
// W2 (core-matrix order) and Wq are staged ONCE per CTA with TMA bulk copies; the A' rows of row group it+2 are
// prefetched into a two-deep ring while it / it+1 are being computed.  The 2 compute warpgroups (128 threads each,
// 2 warps per SM sub-partition, up to 255 registers) are independent pipelines: warpgroup g owns the j-tiles
// [256*jb + 128*g, +128) of every row group, has its own pair-scalar tile, and never waits for the other warpgroup.
// (An optional start-up skew, skew_ns, can de-phase the warpgroups so that their MUFU-idle epilogues fall into
// different time windows; off by default.)
//   * For each hidden chunk of 64 channels and each row i a warp produces the 64 bf16 hidden values of its 32
//     pairs in registers (fp32 math, one MUFU.TANH per value), packed directly in the mma.sync A-fragment layout,
//     and multiplies each 16-channel slab with the W2 slab in shared memory right away (mma.sync m16n8k16, fp32
//     accumulators in registers): the O(N^2 H) hidden tensor never leaves the registers.  H is padded to 16 (one
//     K step), not 64: the last chunk runs 1..4 slabs.  The accumulators of the TI rows (m_pre[i], 32 pairs x 16
//     per warp) stay in registers across all chunks -- 64 per thread, which is why a warpgroup has 255 registers.
//   * After the last chunk the accumulators go through a per-warp shared-memory tile to the thread that owns the
//     pair, which applies SiLU / gate / coors MLP / mask / clamp in fp32; the warp reduces over j with shuffles
//     into per-warp partial sums in shared memory.  The LAST warpgroup to finish a row group (shared-memory
//     counter) adds the partials in a fixed order (deterministic), writes m_i and x_i' once per row, and issues the
//     TMA prefetch of row group it+2 into the ring slot that just became free.
//
// Thread <-> data mappings inside a compute warp:
//   "pair" mapping     (geometry, epilogue): lane l owns pair row 32*wq + l of the tile;
//   "fragment" mapping (hidden production, mma.sync A / D fragments): lane (lr = l/4, lq = l%4) owns rows
//     lr + 8*rho (rho = 0..3) of the warp's 32-row quadrant and, in every 16-channel K-slab, channels
//     4*lq .. 4*lq+3.  Lanes sharing lq read the same A'/Wq words (4 distinct addresses per warp instead
//     of a 32-way broadcast, which cost one shared-memory wavefront per 4 bytes in the first version).
#pragma once

#include <cuda_bf16.h>
#include "common.cuh"
#include "tc_common.cuh"

namespace egnn {

#ifndef EPI_UNROLL
#define EPI_UNROLL 2
#endif
constexpr int TP_EPI_UNROLL = EPI_UNROLL;
constexpr int TP_TI = 4;          // query rows per row group
constexpr int TP_KC = 64;         // hidden channels per chunk (4 K slabs)
constexpr int TP_WG = 2;          // compute warpgroups
constexpr int TP_CWARPS = TP_WG * 4;
constexpr int TP_THREADS = TP_WG * 128;      // 8 warps = 2 per SM sub-partition, up to 255 registers each
constexpr int TP_JB = TP_WG * 128;    // neighbours per block
constexpr int TP_ACC_LD = 18;         // floats per pair row of the per-warp accumulator transpose tile
constexpr int TP_EPI_FLOATS = 64 * 16 + 64 + 64 + 16 + 16 + 4;   // W3 | b3 | w4 | b2 | gate_w | gate_b, b4, scale, 0
constexpr int TP_QMAX = 12;           // per-pair scalar channels of the generic instantiation
constexpr int TP_CMAX = 8;            // coordinate dimensions of the generic instantiation

struct TcPairArgs {
  int B, N, Hp, ldn;               // Hp: H rounded up to 16; ldn: row stride of node_in (bf16 elements)
  int C, Q, F, edge_dim, num_labels;   // Q = 1 + 2F + edge_dim + num_labels  (lean kernel: C = 3, Q = 1)
  int row0, row1;                  // i-rows [row0, row1) of every graph are evaluated (row-sharded multi-GPU)
  uint32_t flags; int has_mask; float clamp;
  uint32_t skew_ns;                // start-up delay between consecutive warpgroups
  int jsplit;                      // j-blocks of a row group are dealt to `jsplit` work items (1 = one item per row group)
  double* gpart;                   // [B * row groups][jsplit][TI][PW] partial sums of the items (jsplit > 1)
  unsigned int* gcount;            // [B * row groups] arrival counters, zero on entry and on exit (jsplit > 1)
  const float* Atab;               // [M][Hp]  0.5 (h W1_i^T + b1)
  const __nv_bfloat16* Btab;       // [M][Hp]  0.5 h W1_j^T
  const float* wq;                 // [Q][Hp]  0.5 * per-pair scalar columns of W1: d | sin | cos | edges | label table
  const __nv_bfloat16* w2p;        // [Hp/16][2][2][8][8]  W2 in core-matrix order
  const float* epi;                // TP_EPI_FLOATS
  const float* coors;              // [B][N][C]
  const __nv_bfloat16* edges;      // [B][N][N][edge_dim] | null
  const uint8_t* labels;           // [B][N][N] | null
  const uint8_t* mask;             // [B][N] | null
  __nv_bfloat16* m_out;            // node_in + dim (stride ldn) | null
  float* coors_out;                // [B][N][C] | null
};

template <bool GEN> struct TpCfg {
  static constexpr int PW = GEN ? 28 : 20;          // partial-sum record per (warp, row): 16 m | C coords | count
  static constexpr int XC = GEN ? TP_CMAX : 4;      // floats per x_i record
};

// Generic instantiation: the per-pair scalar tile keeps d and the fourier features in fp32 (Qf = 1 + 2F planes) and the
// continuous edge channels / one-hot labels in bf16 (Qh planes; both are exactly representable: edges arrive as bf16).
inline size_t tc_pair_gen_scalar_bytes(int Qf, int Qh) { return (size_t)TP_TI * TP_JB * (Qf * 4 + Qh * 2); }

template <bool GEN>
inline size_t tc_pair_smem_bytes(int Hp, int Q, int Qf = 1) {
  size_t n = 0;
  n += (size_t)Hp * 32;                                     // W2 slabs
  n += (size_t)Q * Hp * 4;                                  // Wq
  n += (size_t)2 * TP_TI * Hp * 4;                          // A' rows, two-deep ring
  n += (size_t)TP_EPI_FLOATS * 4;                           // epilogue constants
  n += (size_t)2 * TP_CWARPS * TP_TI * TpCfg<GEN>::PW * 8;  // per-warp partial sums (fp64), per ring slot
  n += (size_t)TP_CWARPS * 32 * TP_ACC_LD * 4;               // per-warp accumulator transpose tile
  n += (size_t)2 * TP_TI * TpCfg<GEN>::XC * 4 + 2 * TP_TI * 4 + 64;   // x_i, mask_i per ring slot; counters, flags
  n += (size_t)(GEN ? 0 : 1) * TP_TI * TP_JB * 4;           // lean: d_ij of the current tiles
  (void)Q;
  if (GEN) n += tc_pair_gen_scalar_bytes(Qf, Q - Qf);
  n += 8 * 8;                                               // mbarriers
  return n + 256;
}

// named barrier over one warpgroup (ids 1..4; id 0 is __syncthreads)
__device__ __forceinline__ void tp_wg_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(g + 1) : "memory"); }

// End of a work item, run by the LAST warpgroup of the CTA to finish it (kept out of line: its registers must not add to the
// pressure of the round loop).  jsplit == 1: add the warps' partial sums and write m_i / x_i'.  jsplit > 1: publish this
// item's sums; the last of the row group's items (device-scope counter) adds the parts in order and writes the outputs.
struct TpFinishArgs {               // the fields of TcPairArgs the finish needs, passed BY VALUE (a reference to the kernel
  int jsplit, N, C, ldn, has_mask;  // parameter block would force a local-memory copy of all of it)
  uint32_t flags;
  double* gpart; unsigned int* gcount; __nv_bfloat16* m_out; float* coors_out;
};
template <bool GEN>
__device__ __noinline__ void tp_finish_item(const TpFinishArgs a, const double* partb, uint32_t* misc, const float* xi, int item, int b,
                                            int i0, int rows_valid, int active_wgs, int g, int t128) {
  constexpr int PW = TpCfg<GEN>::PW, XC = TpCfg<GEN>::XC;
  const int N = a.N, C = a.C;
  const bool upd_feats = a.flags & EGNN_FLAG_UPDATE_FEATS, upd_coors = a.flags & EGNN_FLAG_UPDATE_COORS;
        const int S = a.jsplit;
        const int rgid = item / S;                         // global row-group index
        bool finish = true;                                // does this item write the row group's outputs?
        if (S > 1) {
          // publish this item's sums, then find out whether it is the last of the row group's S items
          if (t128 < TP_TI * PW) {
            const int i = t128 / PW, o = t128 % PW;
            const double* pb = partb + i * PW;
            double sum = 0.0;
            for (int wv = 0; wv < active_wgs * 4; ++wv) sum += pb[(size_t)wv * TP_TI * PW + o];
            a.gpart[(((size_t)rgid * S + (item % S)) * TP_TI + i) * PW + o] = sum;
          }
          __threadfence();
          tp_wg_sync(g);
          if (t128 == 0) {
            const unsigned int old = atomicAdd(&a.gcount[rgid], 1u);
            if (old == (unsigned)S - 1) a.gcount[rgid] = 0;          // ready for the next launch
            __threadfence();
            misc[8 + g] = (old == (unsigned)S - 1);
          }
          tp_wg_sync(g);
          finish = misc[8 + g] != 0;
        }
        if (finish && t128 < TP_TI * (PW - 1)) {
          const int i = t128 / (PW - 1), o = t128 % (PW - 1);
          if (i < rows_valid) {
            const double* pb = partb + i * PW;
            double s = 0.0, cnt = 0.0;
            if (S > 1) {
              for (int pp = 0; pp < S; ++pp) {
                const double* gp = a.gpart + (((size_t)rgid * S + pp) * TP_TI + i) * PW;
                s += __ldcg(gp + o);
                cnt += __ldcg(gp + PW - 1);
              }
            } else {
#pragma unroll
              for (int wv = 0; wv < TP_CWARPS; ++wv)
                if (wv < active_wgs * 4) s += pb[(size_t)wv * TP_TI * PW + o];      // idle warpgroups never wrote theirs
              for (int wv = 0; wv < active_wgs * 4; ++wv) cnt += pb[(size_t)wv * TP_TI * PW + PW - 1];
            }
            const size_t node = (size_t)b * N + i0 + i;
            if (o < 16) {
              if (upd_feats) {
                float inv = 1.f;
                if (a.flags & EGNN_FLAG_POOL_MEAN) inv = a.has_mask ? (cnt > 0.0 ? 1.f / (float)cnt : 0.f) : 1.f / (float)N;   // :325-330
                a.m_out[node * a.ldn + o] = __float2bfloat16((float)s * inv);
              }
            } else if (o - 16 < C) {
              if (upd_coors) a.coors_out[node * C + (o - 16)] = xi[i * XC + (o - 16)] + (float)s;             // :315
            }
          }
        }
}

template <bool GEN>
__global__ void __launch_bounds__(TP_THREADS, 1) tc_pair_kernel(const TcPairArgs a) {
  constexpr int PW = TpCfg<GEN>::PW, XC = TpCfg<GEN>::XC;
  // carve the dynamic shared memory directly (no integer round trip) so every access stays in the
  // shared state space (LDS/STS, not generic LD/ST); nothing here needs more than 128-byte alignment
  extern __shared__ __align__(128) unsigned char sm[];
  const int Hp = a.Hp, N = a.N;
  const int Q = GEN ? a.Q : 1, C = GEN ? a.C : 3;
  unsigned char* w2s = sm;                                                    // Hp*32 bytes
  float* wqs = reinterpret_cast<float*>(w2s + (size_t)Hp * 32);               // [Q][Hp]
  float* As = wqs + (size_t)Q * Hp;                                           // [2][TI][Hp]
  float* epi = As + (size_t)2 * TP_TI * Hp;                                   // constants
  // Sums ACROSS tiles are kept in fp64: the per-tile sums are fp32 (fixed shuffle tree), and adding a few hundred
  // fp32 numbers in fp64 is exact, so the result does not depend on how the tiles were dealt to warps, work items or
  // ranks (row-sharded == single GPU, bit for bit, whatever jsplit is).
  double* part = reinterpret_cast<double*>(epi + TP_EPI_FLOATS);              // [2][CWARPS][TI][PW]
  float* xis = reinterpret_cast<float*>(part + 2 * TP_CWARPS * TP_TI * PW);   // [2][TI][XC]
  uint32_t* mki = reinterpret_cast<uint32_t*>(xis + 2 * TP_TI * XC);          // [2][TI]
  uint32_t* misc = mki + 2 * TP_TI;                                           // [0..1] done counters, [4..] last flags
  const int Qf = GEN ? 1 + 2 * a.F : 1, Qh = Q - Qf;
  float* ssm = reinterpret_cast<float*>(misc + 16);                           // [WG][Qf][TI][128] fp32
  __nv_bfloat16* ssh = reinterpret_cast<__nv_bfloat16*>(ssm + (size_t)Qf * TP_TI * TP_JB);   // [WG][Qh][TI][128] bf16
  float* accs = reinterpret_cast<float*>(ssh + (size_t)Qh * TP_TI * TP_JB);    // [CWARPS][32][TP_ACC_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(accs + TP_CWARPS * 32 * TP_ACC_LD);
  uint64_t* ldbar = bars;                         // W2 / Wq staging
  uint64_t* rowfull = ldbar + 1;                  // [2] A' ring

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rows_per_graph = a.row1 - a.row0;
  const int rg_per_graph = (rows_per_graph + TP_TI - 1) / TP_TI;
  // Work items: (graph, row group, j part).  With few row groups per SM (row-sharded graphs, small batches) a row
  // group's j-blocks are dealt round-robin to S = jsplit items so that the static schedule has enough items to balance;
  // the S partial sums of a row group meet in global memory and the LAST item to arrive (device-scope counter) adds them
  // in part order -- deterministic -- and writes the outputs.
  const int n_items = a.B * rg_per_graph * a.jsplit;          // (jsplit >= 1, set by the launcher)
  const int nchunks = (Hp + TP_KC - 1) / TP_KC;
  const int nsl_last = (Hp - (nchunks - 1) * TP_KC) / 16;        // valid K slabs of the last chunk, 1..4
  const int njb = (N + TP_JB - 1) / TP_JB;
  const bool upd_feats = a.flags & EGNN_FLAG_UPDATE_FEATS, upd_coors = a.flags & EGNN_FLAG_UPDATE_COORS;

  auto item_rows = [&](int item, int& b, int& i0, int& rows_valid) {
    item /= a.jsplit;                                                // (the j part is item % jsplit)
    b = item / rg_per_graph;
    i0 = a.row0 + (item - b * rg_per_graph) * TP_TI;
    rows_valid = min(TP_TI, a.row1 - i0);
  };
  // Stage the per-row-group data of `item` into ring slot `buf`.  Called by 128 threads (rank t = 0..127) that can
  // synchronise with `sync()`: x_i / mask_i by plain stores from TI*XC (+TI) of them in parallel, then ONE thread
  // arms the rowfull barrier (the stores become visible to the consumers through its release/acquire) and issues
  // the TMA bulk copy of the A' rows.
  auto stage_item = [&](int item, int buf, int t, auto sync) {
    int b, i0, rows_valid;
    item_rows(item, b, i0, rows_valid);
    if (t < TP_TI * XC) {
      const int r = t / XC, c = t % XC;
      const size_t node = (size_t)b * N + (r < rows_valid ? i0 + r : i0);
      xis[(buf * TP_TI + r) * XC + c] = c < C ? a.coors[node * C + c] : 0.f;
    } else if (t < TP_TI * XC + TP_TI) {
      const int r = t - TP_TI * XC;
      const size_t node = (size_t)b * N + (r < rows_valid ? i0 + r : i0);
      mki[buf * TP_TI + r] = (r < rows_valid) && (a.has_mask ? a.mask[node] != 0 : true);
    }
    sync();
    if (t == 0) {
      const uint32_t bytes = (uint32_t)rows_valid * Hp * 4;
      tc::mbar_arrive_expect_tx(&rowfull[buf], bytes);
      const unsigned char* src = reinterpret_cast<const unsigned char*>(a.Atab + ((size_t)b * N + i0) * Hp);
      const uint32_t dst = tc::smem_u32(As + (size_t)buf * TP_TI * Hp);
      for (uint32_t o = 0; o < bytes; o += 16384) tc::tma_bulk_g2s(dst + o, src + o, min(16384u, bytes - o), &rowfull[buf]);
    }
  };

  // ---------------- setup
  if (tid == 0) {
    tc::mbar_init(ldbar, 1);
    tc::mbar_init(&rowfull[0], 1); tc::mbar_init(&rowfull[1], 1);
    tc::mbar_fence_init();
  }
  for (int x = tid; x < TP_EPI_FLOATS; x += TP_THREADS) epi[x] = a.epi[x];
  for (int x = tid; x < 2 * TP_TI * Hp; x += TP_THREADS) As[x] = 0.f;      // rows beyond a graph's end stay finite
  if (tid < 2) misc[tid] = 0;
  tc::fence_proxy_async_smem();                    // the zero fill above precedes TMA writes to the same buffers
  __syncthreads();

  if (tid == 0) {
    // TMA bulk staging, once per CTA: W2 slabs and the per-pair scalar columns
    const uint32_t w2_bytes = (uint32_t)Hp * 32, wq_bytes = (uint32_t)Q * Hp * 4;
    tc::mbar_arrive_expect_tx(ldbar, w2_bytes + wq_bytes);
    auto bulk = [&](uint32_t dst, const unsigned char* src, uint32_t bytes) {
      for (uint32_t o = 0; o < bytes; o += 16384) tc::tma_bulk_g2s(dst + o, src + o, min(16384u, bytes - o), ldbar);
    };
    bulk(tc::smem_u32(w2s), reinterpret_cast<const unsigned char*>(a.w2p), w2_bytes);
    bulk(tc::smem_u32(wqs), reinterpret_cast<const unsigned char*>(a.wq), wq_bytes);
  }
  if (warp < 4) {                                  // warpgroup 0 stages the first two row groups of this CTA
    auto sync0 = [&]() { tp_wg_sync(0); };
    if ((int)blockIdx.x < n_items) stage_item(blockIdx.x, 0, tid, sync0);
    if ((int)(blockIdx.x + gridDim.x) < n_items) stage_item(blockIdx.x + gridDim.x, 1, tid, sync0);
  }

  {
    // =========================================================== compute warpgroups (independent pipelines)
    const int g = warp >> 2, wq = warp & 3, t128 = tid & 127;
    const int lr = lane >> 2, lq = lane & 3;
    float* swg = ssm + (size_t)g * Qf * TP_TI * 128;  // pair scalars of this warpgroup's tile: swg[(q*TI + i)*128 + pair]
    __nv_bfloat16* shg = ssh + (size_t)g * Qh * TP_TI * 128;
    float* myacc = accs + (size_t)warp * 32 * TP_ACC_LD;
    if (a.skew_ns && g > 0) {                         // de-phase the warpgroups (see the header)
      uint64_t t0, t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      const uint64_t until = t0 + (uint64_t)a.skew_ns * g;
      do { __nanosleep(1000); asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 < until);
    }
    // warpgroups whose j-tiles all lie beyond the graph (N <= 128 g) have nothing to do in ANY row group: they leave
    // now instead of spinning on the ring barriers next to the working warps of their SM sub-partitions
    const int active_wgs = min(TP_WG, (N + 127) / 128);
    const bool wg_active = g < active_wgs;
    if (wg_active) tc::mbar_wait(ldbar, 0);
    int it = 0;
    for (int item = blockIdx.x; wg_active && item < n_items; item += gridDim.x, ++it) {
      const int buf = it & 1;
      int b, i0, rows_valid;
      item_rows(item, b, i0, rows_valid);
      tc::mbar_wait(&rowfull[buf], (it >> 1) & 1);
      const float* Ab = As + (size_t)buf * TP_TI * Hp;
      const float* xi = xis + buf * TP_TI * XC;
      const uint32_t* mk = mki + buf * TP_TI;
      double* mypart = part + ((size_t)buf * TP_CWARPS + warp) * TP_TI * PW;
      for (int x = lane; x < TP_TI * PW; x += 32) mypart[x] = 0.0;
      __syncwarp();

      for (int jb = item % a.jsplit; jb < njb; jb += a.jsplit) {
        if (jb * TP_JB + g * 128 >= N) break;           // this warpgroup's tile lies beyond the graph
        // ---- pair mapping: geometry (and the other per-pair scalar channels) of (i, j) for the rows i
        const int j = jb * TP_JB + g * 128 + t128;
        const bool jv = j < N;
        const size_t nodej = (size_t)b * N + (jv ? j : N - 1);
        float xj[GEN ? TP_CMAX : 3];
#pragma unroll
        for (int c = 0; c < (GEN ? TP_CMAX : 3); ++c) xj[c] = (!GEN || c < C) ? a.coors[nodej * C + c] : 0.f;
        const bool mask_j = jv && (a.has_mask ? a.mask[nodej] != 0 : true);
        __syncwarp();                                   // previous tile's readers of swg are done
#pragma unroll
        for (int i = 0; i < TP_TI; ++i) {
          float d = 0.f;
#pragma unroll
          for (int c = 0; c < (GEN ? TP_CMAX : 3); ++c) { const float r = xi[i * XC + c] - xj[c]; d = fmaf(r, r, d); }
          swg[i * 128 + t128] = d;
          if (GEN) {
            int q = 1;
            for (int f = 0; f < a.F; ++f) {                                                       // :34-41
              const float sc = d * exp2f(-(float)f);
              swg[((q + f) * TP_TI + i) * 128 + t128] = sinf(sc);
              swg[((q + a.F + f) * TP_TI + i) * 128 + t128] = cosf(sc);
            }
            const size_t pij = ((size_t)b * N + min(i0 + i, N - 1)) * N + (jv ? j : N - 1);
            for (int e = 0; e < a.edge_dim; ++e) shg[(e * TP_TI + i) * 128 + t128] = a.edges[pij * a.edge_dim + e];
            if (a.num_labels > 0) {
              const int lab = a.labels[pij];
              for (int l = 0; l < a.num_labels; ++l)
                shg[((a.edge_dim + l) * TP_TI + i) * 128 + t128] = __float2bfloat16((l == lab) ? 1.f : 0.f);
            }
          }
        }
        __syncwarp();
        // ---- fragment mapping: B' rows of this lane's 4 pairs
        // (rows lr + 8 rho of the tile are 8 table rows apart: one base pointer + a stride instead of four pointers.  Rows
        //  beyond the graph are NOT clamped: they read the next graph's rows or the 128 padding rows of the table, and
        //  their pairs are discarded by `jv` -- NaN-safe, every use is a select)
        const uint2* Bp0 = reinterpret_cast<const uint2*>(a.Btab + ((size_t)b * N + jb * TP_JB + g * 128 + wq * 32 + lr) * Hp + 4 * lq);
        const int Bstride = 8 * Hp / 4;                 // uint2 units between rows lr + 8 rho and lr + 8 (rho + 1)
#define Bp_(rho) (Bp0 + (rho) * Bstride)
        uint2 Bc[4][4];                                 // [rho][slab] B' of the current chunk (bf16 x4 each)
        {
          const int nsl0 = nchunks == 1 ? nsl_last : 4;
#pragma unroll
          for (int rho = 0; rho < 4; ++rho)
#pragma unroll
            for (int sl = 0; sl < 4; ++sl) Bc[rho][sl] = sl < nsl0 ? __ldg(Bp_(rho) + sl * 4) : make_uint2(0u, 0u);
        }

        float acc[TP_TI][2][2][4];                      // m_pre[i] of rows [16 half, +16) x channels [8 nt, +8) (D fragments)
#pragma unroll
        for (int i = 0; i < TP_TI; ++i)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int e = 0; e < 4; ++e) acc[i][h][nt][e] = 0.f;
        // A chunk with all 4 K slabs runs with NSLC = 4 (every slab test folds at compile time); only the last chunk
        // of a hidden width that is not a multiple of 64 takes the predicated instantiation (NSLC = 0).
        auto chunk = [&](const int c, auto nslc) {
          constexpr int NSLC = decltype(nslc)::value;
          const int nsl = NSLC ? NSLC : nsl_last;                   // valid slabs of this chunk
          const int nsl_next = c + 2 == nchunks ? nsl_last : 4;     // ... and of the next one (prefetch)
          // Register budget: w_d and A' are read from shared memory at the point of use instead of being held for the chunk
          // / round; one B' base pointer + stride; every slab is multiplied as soon as it is packed.
          // One round = the 64 hidden channels of chunk c for row i and this warp's 32 pairs.  In the last round
          // of a chunk (`reload`), every B' register is re-filled for chunk c+1 right after its last use, so the
          // L2 latency is covered by the rest of that round without a second register buffer.
          // The row index is a compile-time constant (IntC) so that acc[i] stays in registers.
          auto round = [&](auto i_tag, auto reload_tag) {
            constexpr int i = decltype(i_tag)::value;
            constexpr bool reload = decltype(reload_tag)::value != 0;
            const float* Ai = Ab + (size_t)i * Hp + c * TP_KC + lq * 4;
            float dr[4];
            if (!GEN) {
#pragma unroll
              for (int rho = 0; rho < 4; ++rho) dr[rho] = swg[i * 128 + wq * 32 + lr + 8 * rho];
            }
#pragma unroll
            for (int half = 0; half < 2; ++half) {       // rows (lr, lr+8), then (lr+16, lr+24)
              // GEN: z = A' + sum_q Wq s_q (pre-activation / 2 without B') for 2 pairs x 16 channels, q outermost
              float2 z[GEN ? 4 : 1][2][2];               // [slab][r2][channel pair]
              if (GEN) {
#pragma unroll
                for (int sl = 0; sl < 4; ++sl) {
                  const float4 av = sl < nsl ? *reinterpret_cast<const float4*>(Ai + sl * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                  for (int r2 = 0; r2 < 2; ++r2) {
                    z[GEN ? sl : 0][r2][0] = make_float2(av.x, av.y);
                    z[GEN ? sl : 0][r2][1] = make_float2(av.z, av.w);
                  }
                }
#pragma unroll 1
                for (int q = 0; q < Q; ++q) {
                  float s0, s1;
                  if (q < Qf) {
                    const float* sq = swg + (q * TP_TI + i) * 128 + wq * 32 + lr + 16 * half;
                    s0 = sq[0]; s1 = sq[8];
                  } else {
                    const __nv_bfloat16* sq = shg + ((q - Qf) * TP_TI + i) * 128 + wq * 32 + lr + 16 * half;
                    s0 = __bfloat162float(sq[0]); s1 = __bfloat162float(sq[8]);
                  }
                  const float2 ss0 = make_float2(s0, s0), ss1 = make_float2(s1, s1);
                  const float* wrow = wqs + (size_t)q * Hp + c * TP_KC + lq * 4;
#pragma unroll
                  for (int sl = 0; sl < 4; ++sl) {
                    if (sl < nsl) {
                      const float4 wv = *reinterpret_cast<const float4*>(wrow + sl * 16);
                      float2 (&zz)[2][2] = z[GEN ? sl : 0];
                      zz[0][0] = tc::ffma2(make_float2(wv.x, wv.y), ss0, zz[0][0]);
                      zz[0][1] = tc::ffma2(make_float2(wv.z, wv.w), ss0, zz[0][1]);
                      zz[1][0] = tc::ffma2(make_float2(wv.x, wv.y), ss1, zz[1][0]);
                      zz[1][1] = tc::ffma2(make_float2(wv.z, wv.w), ss1, zz[1][1]);
                    }
                  }
                }
              }
              uint32_t hp[16];
#pragma unroll
              for (int sl = 0; sl < 4; ++sl) {
                if (NSLC == 0 && sl >= nsl) continue;      // tail chunk: slabs beyond H are neither computed nor multiplied
#pragma unroll
                for (int r2 = 0; r2 < 2; ++r2) {
                  const int rho = half * 2 + r2;
                  const uint2 bb = Bc[rho][sl];
                  float2 z01, z23;
                  if (GEN) {
                    z01 = z[GEN ? sl : 0][r2][0]; z23 = z[GEN ? sl : 0][r2][1];
                  } else {
                    const float4 av = *reinterpret_cast<const float4*>(Ai + sl * 16);
                    const float d = dr[rho];
                    const float2 dd = make_float2(d, d);
                    const float4 wv = *reinterpret_cast<const float4*>(wqs + c * TP_KC + sl * 16 + lq * 4);
                    z01 = tc::ffma2(make_float2(wv.x, wv.y), dd, make_float2(av.x, av.y));   // wd*d + A'
                    z23 = tc::ffma2(make_float2(wv.z, wv.w), dd, make_float2(av.z, av.w));
                  }
                  const float2 y01 = make_float2(tc::add_bf16_lo(bb.x, z01.x), tc::add_bf16_hi(bb.x, z01.y));  // + B'
                  const float2 y23 = make_float2(tc::add_bf16_lo(bb.y, z23.x), tc::add_bf16_hi(bb.y, z23.y));
                  const float2 h01 = tc::ffma2(y01, make_float2(tc::tanh_fast(y01.x), tc::tanh_fast(y01.y)), y01);  // y + y tanh y
                  const float2 h23 = tc::ffma2(y23, make_float2(tc::tanh_fast(y23.x), tc::tanh_fast(y23.y)), y23);
                  // A fragment: regs {0,1} of a slab -> row lr (+16), regs {2,3} -> row lr+8 (+24); even k low
                  hp[sl * 4 + r2 * 2 + 0] = tc::pack_bf16x2(h01.x, h01.y);
                  hp[sl * 4 + r2 * 2 + 1] = tc::pack_bf16x2(h23.x, h23.y);
                  if (reload && sl < nsl_next) Bc[rho][sl] = __ldg(Bp_(rho) + (c + 1) * 16 + sl * 4);
                }
                const uint32_t h4[4] = {hp[sl * 4], hp[sl * 4 + 1], hp[sl * 4 + 2], hp[sl * 4 + 3]};
                tc::mma_w2_slab(acc[i][half], h4, w2s, c * 4 + sl, lr, lq);
              }
            }
          };
          static_assert(TP_TI == 4, "the rounds of a chunk are spelled out below");
          round(tc::IntC<0>{}, tc::IntC<0>{});
          round(tc::IntC<1>{}, tc::IntC<0>{});
          round(tc::IntC<2>{}, tc::IntC<0>{});
          // the last round of a full chunk re-fills B' for the next chunk; the tail chunk is always the last one
          if (NSLC != 0 && c + 1 < nchunks) round(tc::IntC<3>{}, tc::IntC<1>{});
          else round(tc::IntC<3>{}, tc::IntC<0>{});
        };
        {
          const int nfull = nsl_last == 4 ? nchunks : nchunks - 1;
#pragma unroll 1
          for (int c = 0; c < nfull; ++c) chunk(c, tc::IntC<4>{});
          if (nfull < nchunks) chunk(nchunks - 1, tc::IntC<0>{});
        }

        // ---- epilogue of this tile: accumulators back to the owning thread (pair mapping)
        const float* W3 = epi; const float* b3 = epi + 1024; const float* w4 = b3 + 64;
        const float* b2 = w4 + 64; const float* gw = b2 + 16; const float* sc = gw + 16;   // sc: gate_b, b4, scale
        float m[TP_TI][16];                              // m_ij of this thread's pair for the TI rows
#pragma unroll
        for (int i = 0; i < TP_TI; ++i) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int r2 = 0; r2 < 2; ++r2)
                *reinterpret_cast<float2*>(myacc + (16 * h + 8 * r2 + lr) * TP_ACC_LD + 8 * nt + 2 * lq) =
                    make_float2(acc[i][h][nt][2 * r2], acc[i][h][nt][2 * r2 + 1]);
          __syncwarp();
#pragma unroll
          for (int o = 0; o < 16; ++o) m[i][o] = tc::silu_half_arg(0.5f * (myacc[lane * TP_ACC_LD + o] + b2[o]));    // :183
          __syncwarp();
          if (a.flags & EGNN_FLAG_SOFT_EDGES) {                                                               // :289-290
            float z = sc[0];
#pragma unroll
            for (int o = 0; o < 16; ++o) z = fmaf(gw[o], m[i][o], z);
            const float gate = 0.5f + 0.5f * tc::tanh_fast(0.5f * z);
#pragma unroll
            for (int o = 0; o < 16; ++o) m[i][o] *= gate;
          }
        }
        float wgt[TP_TI];
#pragma unroll
        for (int i = 0; i < TP_TI; ++i) wgt[i] = 0.f;
        if (upd_coors) {                                                                                      // :302-315
          // hidden unit u outermost: one W3 row (4 x LDS.128) serves all TI rows of this pair; the four rows are four
          // independent FMA chains
#pragma unroll TP_EPI_UNROLL
          for (int u = 0; u < 64; ++u) {
            const float4* w3 = reinterpret_cast<const float4*>(W3 + u * 16);
            const float4 wa = w3[0], wb = w3[1], wc = w3[2], wd4 = w3[3];
            const float bu = b3[u], w4u = w4[u];
#pragma unroll
            for (int i = 0; i < TP_TI; ++i) {
              float tt = bu;
              tt = fmaf(wa.x, m[i][0], tt); tt = fmaf(wa.y, m[i][1], tt); tt = fmaf(wa.z, m[i][2], tt); tt = fmaf(wa.w, m[i][3], tt);
              tt = fmaf(wb.x, m[i][4], tt); tt = fmaf(wb.y, m[i][5], tt); tt = fmaf(wb.z, m[i][6], tt); tt = fmaf(wb.w, m[i][7], tt);
              tt = fmaf(wc.x, m[i][8], tt); tt = fmaf(wc.y, m[i][9], tt); tt = fmaf(wc.z, m[i][10], tt); tt = fmaf(wc.w, m[i][11], tt);
              tt = fmaf(wd4.x, m[i][12], tt); tt = fmaf(wd4.y, m[i][13], tt); tt = fmaf(wd4.z, m[i][14], tt); tt = fmaf(wd4.w, m[i][15], tt);
              wgt[i] = fmaf(w4u, tc::silu_half_arg(0.5f * tt), wgt[i]);
            }
          }
        }
#pragma unroll
        for (int i = 0; i < TP_TI; ++i) {
          const bool pm = jv && (mk[i] != 0) && (a.has_mask ? mask_j : true);
          float w = wgt[i] + sc[1];
          if (upd_coors) {
            if (!pm) w = 0.f;                                                                                 // :309
            if (a.flags & EGNN_FLAG_CLAMP) w = fminf(fmaxf(w, -a.clamp), a.clamp);                            // :313
            if (a.flags & EGNN_FLAG_NORM_COORS) w *= sc[2] / fmaxf(sqrtf(swg[i * 128 + t128]), 1e-8f);        // :74-77
          } else {
            w = 0.f;
          }
          float v[PW];
#pragma unroll
          for (int o = 0; o < 16; ++o) v[o] = pm ? m[i][o] : 0.f;                                             // :322
#pragma unroll
          for (int c = 0; c < PW - 17; ++c) {
            constexpr int NX = GEN ? TP_CMAX : 3;
            v[16 + c] = (c < NX && (!GEN || c < C)) ? w * (xi[i * XC + (c < NX ? c : 0)] - xj[c < NX ? c : 0]) : 0.f;
          }
          v[PW - 1] = pm ? 1.f : 0.f;
#pragma unroll
          for (int off = 16; off > 0; off >>= 1)
#pragma unroll
            for (int o = 0; o < PW; ++o) v[o] += __shfl_xor_sync(0xffffffffu, v[o], off);
          if (lane == 0) {
#pragma unroll
            for (int o = 0; o < PW; ++o) mypart[i * PW + o] += (double)v[o];
          }
        }
      }

      // ---- this warpgroup is done with the row group: the last of the four finishes it
      __syncwarp();
      tp_wg_sync(g);                                       // all partial sums of this warpgroup are in shared memory
      if (t128 == 0) {
        __threadfence_block();
        const uint32_t old = atomicAdd(&misc[buf], 1u);
        if ((int)old == active_wgs - 1) misc[buf] = 0;     // nobody touches the counter again before the next refill
        __threadfence_block();
        misc[4 + g] = ((int)old == active_wgs - 1);
      }
      tp_wg_sync(g);
      if (misc[4 + g]) {
        TpFinishArgs fa;
        fa.jsplit = a.jsplit; fa.N = N; fa.C = C; fa.ldn = a.ldn; fa.has_mask = a.has_mask; fa.flags = a.flags;
        fa.gpart = a.gpart; fa.gcount = a.gcount; fa.m_out = a.m_out; fa.coors_out = a.coors_out;
        tp_finish_item<GEN>(fa, part + (size_t)buf * TP_CWARPS * TP_TI * PW, misc, xi, item, b, i0, rows_valid, active_wgs, g, t128);
        tp_wg_sync(g);                                     // every reader of ring slot `buf` is done
        const int nxt = item + 2 * gridDim.x;
        if (nxt < n_items) stage_item(nxt, buf, t128, [&]() { tp_wg_sync(g); });
      }
    }
  }

}

}  // namespace egnn

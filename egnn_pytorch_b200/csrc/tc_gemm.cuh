// wgmma GEMM for the per-node contractions of the layer (bf16 operands, fp32 accumulation in registers):
//     out[r, n] = act( scale * (sum_k A[r,k] W[n,k] + bias[n]) ) + R[r, n]
// used for  A' = 0.5 (h W1_i^T + b1)  (fp32 out),  B' = 0.5 h W1_j^T  (bf16 out)   [split of egnn_pytorch.py:287]
//           h1 = SiLU([LN(h) | m_i] Wn1^T + bn1),  h' = h1 Wn2^T + bn2 + h                   [egnn_pytorch.py:335-337]
//
// 128x128 output tile per CTA (one warpgroup), BK = 64, a three-stage shared-memory ring filled with cp.async straight
// into the wgmma swizzle-128B K-major layout (128-byte rows, 8-row groups); per stage the warpgroup issues
// wgmma (M=64, N=128, K=16) x 2 row halves x 4, accumulating in registers (2 x 64 fp32 per thread).
#pragma once

#include <cuda_bf16.h>
#include "tc_common.cuh"

namespace egnn {

struct TcGemmArgs {
  const __nv_bfloat16* A; int lda;    // [M][K]
  const __nv_bfloat16* W; int ldw;    // [Nv][K]
  const float* bias;                  // [Nv] | null
  const __nv_bfloat16* R; int ldr;    // residual [M][Nv] | null
  void* out; int ldo; int out_f32;
  int M, Nv, Nout, K;
  float scale; int act;               // act: 0 none, 1 SiLU
};

constexpr int GEMM_BM = 128, GEMM_BN = 128, GEMM_BK = 64;
constexpr int GEMM_TILE_BYTES = GEMM_BM * GEMM_BK * 2;            // 16 KB per operand per stage (128 rows x 128 B)
constexpr int GEMM_STAGES = 3;   // shared-memory ring (3 x 32 KB: two CTAs per SM, one tile's epilogue overlaps the other's main loop)
constexpr int GEMM_DIST = 2;     // copies run 2 k-steps ahead of the MMAs
constexpr int GEMM_SMEM_BYTES = GEMM_STAGES * 2 * GEMM_TILE_BYTES + 1024;

// Two problems that share nothing but the launch (the A' and B' tables of a layer: same activations, different weight
// blocks, bias and output type): CTAs with blockIdx.x < nt0 work on p[0], the others on p[1].
struct TcGemmPair { TcGemmArgs p[2]; int nt0; };

__global__ void __launch_bounds__(128, 1) tc_gemm_kernel(const TcGemmPair gp) {
  const bool second = (int)blockIdx.x >= gp.nt0;
  // field-wise select (a dynamically indexed kernel-parameter struct would be copied to local memory)
  TcGemmArgs g;
  g.A = second ? gp.p[1].A : gp.p[0].A; g.lda = second ? gp.p[1].lda : gp.p[0].lda;
  g.W = second ? gp.p[1].W : gp.p[0].W; g.ldw = second ? gp.p[1].ldw : gp.p[0].ldw;
  g.bias = second ? gp.p[1].bias : gp.p[0].bias;
  g.R = second ? gp.p[1].R : gp.p[0].R; g.ldr = second ? gp.p[1].ldr : gp.p[0].ldr;
  g.out = second ? gp.p[1].out : gp.p[0].out; g.ldo = second ? gp.p[1].ldo : gp.p[0].ldo;
  g.out_f32 = second ? gp.p[1].out_f32 : gp.p[0].out_f32;
  g.M = second ? gp.p[1].M : gp.p[0].M; g.Nv = second ? gp.p[1].Nv : gp.p[0].Nv; g.Nout = second ? gp.p[1].Nout : gp.p[0].Nout;
  g.K = second ? gp.p[1].K : gp.p[0].K; g.scale = second ? gp.p[1].scale : gp.p[0].scale; g.act = second ? gp.p[1].act : gp.p[0].act;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * GEMM_BM, n0 = ((int)blockIdx.x - (second ? gp.nt0 : 0)) * GEMM_BN;
  const uint32_t s_base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;       // swizzle-128B tiles need 1024-byte alignment
  unsigned char* smem = smem_raw + (s_base - tc::smem_u32(smem_raw));

  const int nk = (g.K + GEMM_BK - 1) / GEMM_BK;
  // Copy mapping: 8 consecutive lanes fetch the 8 16-byte K-chunks of one row (one fully used 128-byte line per
  // row) and drop them into the row's 128 bytes of the swizzle-128B layout (chunk kc -> position kc ^ (row % 8)):
  // coalesced on the global side, conflict-free on the shared side.
  auto load_stage = [&](int kt) {
    const int st = kt % GEMM_STAGES;
    const uint32_t sA = s_base + st * 2 * GEMM_TILE_BYTES, sW = sA + GEMM_TILE_BYTES;
    const int kc = tid & 7, k = kt * GEMM_BK + kc * 8;
    const bool kin = k < g.K;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int r = it * 16 + (tid >> 3);
      const int rowA = m0 + r, rowW = n0 + r;
      const bool va = kin && rowA < g.M, vw = kin && rowW < g.Nv;
      const __nv_bfloat16* pa = va ? g.A + (size_t)rowA * g.lda + k : g.A;
      const __nv_bfloat16* pw = vw ? g.W + (size_t)rowW * g.ldw + k : g.W;
      const uint32_t off = (uint32_t)r * 128u + (uint32_t)((kc ^ (r & 7)) << 4);
      tc::cp_async16(sA + off, pa, va ? 16u : 0u);
      tc::cp_async16(sW + off, pw, vw ? 16u : 0u);
    }
  };

  // Multi-stage ring.  Every thread copies its rows of stage kt+DIST, waits for its own copies of stage kt
  // (cp.async.wait_group) and makes them visible to the tensor core (fence.proxy.async); after a barrier the
  // warpgroup issues the stage's wgmma (rows 0..63 and 64..127 of the tile, K=16 x 4).  It then waits only for the
  // PREVIOUS k-step's wgmma (wait_group 1) -- the last reader of slot (kt+DIST) % STAGES -- and, after a barrier that
  // makes that true for every warp, refills the slot: the wgmma of stage kt keep running through the refill, the
  // copy wait and the barrier of the next k-step.
  float acc[2][64];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r = 0; r < 64; ++r) acc[h][r] = 0.f;
  for (int kt = 0; kt < GEMM_DIST; ++kt) {
    if (kt < nk) load_stage(kt);
    tc::cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    tc::cp_async_wait<GEMM_DIST - 1>();    // this thread's copies of stage kt have landed
    tc::fence_proxy_async_smem();          // cp.async (generic proxy) -> tensor core (async proxy)
    __syncthreads();
    const uint32_t sA = s_base + (kt % GEMM_STAGES) * 2 * GEMM_TILE_BYTES, sW = sA + GEMM_TILE_BYTES;
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < GEMM_BK / 16; ++kk) {
      const uint64_t dw = tc::wgmma_desc_kmajor_sw128(sW + kk * 32);   // K=16 step = 32 B inside the swizzle atom
#pragma unroll
      for (int h = 0; h < 2; ++h)                                      // rows 64 h .. 64 h + 63: 8 row groups of 1024 B
        tc::wgmma_m64n128k16_ss(acc[h], tc::wgmma_desc_kmajor_sw128(sA + h * 8192 + kk * 32), dw, 1u);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<1>();                   // the wgmma of k-step kt-1 are done (this warp) ...
    __syncthreads();                       // ... and every warp's: slot (kt+DIST) % STAGES is free
    const int nxt = kt + GEMM_DIST;
    if (nxt < nk) load_stage(nxt);
    tc::cp_async_commit();
  }
  tc::wgmma_wait<0>();
  __syncthreads();                         // every warp's wgmma are done: the ring is free for the epilogue

  // Epilogue.  The accumulator fragments are spread over the warpgroup (see wgmma_m64n128k16_ss); they go through
  // shared memory (the pipeline buffers are free now) so that each warp then writes its 32 rows with lane = column:
  // 128-byte (fp32) / 64-byte (bf16) contiguous stores, bias and residual loaded once per column / coalesced.
  constexpr int LDS = GEMM_BN + 4;
  float* stg = reinterpret_cast<float*>(smem);                    // [128][LDS]
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r = 0; r < 64; r += 2) {
      const int row = 64 * h + 16 * warp + (lane >> 2) + 8 * ((r >> 1) & 1), col = 8 * (r >> 2) + 2 * (lane & 3);
      *reinterpret_cast<float2*>(stg + row * LDS + col) = make_float2(acc[h][r], acc[h][r + 1]);
    }
  __syncthreads();
#pragma unroll 1
  for (int cb = 0; cb < GEMM_BN / 32; ++cb) {
    const int col0 = n0 + cb * 32;
    if (col0 >= g.Nout) break;
    const int col = col0 + lane;
    const bool cin = col < g.Nout, cv = col < g.Nv;
    const float bcol = (cv && g.bias) ? g.bias[col] : 0.f;
    // residual rows: all 32 loads are issued before the first one is consumed (one dependent global load per row
    // makes the residual GEMM latency-bound)
    __nv_bfloat16 rres[32];
    if (g.R) {
#pragma unroll
      for (int rr = 0; rr < 32; ++rr) {
        const int row = m0 + warp * 32 + rr;
        rres[rr] = (cv && row < g.M) ? g.R[(size_t)row * g.ldr + col] : __float2bfloat16(0.f);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 32; ++rr) {
      const int row = m0 + warp * 32 + rr;
      if (row >= g.M) break;
      float x = 0.f;
      if (cv) {
        x = (stg[(warp * 32 + rr) * LDS + cb * 32 + lane] + bcol) * g.scale;
        if (g.act == 1) x = __fdividef(x, 1.0f + __expf(-x));
        if (g.R) x += __bfloat162float(rres[rr]);
      }
      if (cin) {
        if (g.out_f32) static_cast<float*>(g.out)[(size_t)row * g.ldo + col] = x;
        else static_cast<__nv_bfloat16*>(g.out)[(size_t)row * g.ldo + col] = __float2bfloat16(x);
      }
    }
  }
}

}  // namespace egnn

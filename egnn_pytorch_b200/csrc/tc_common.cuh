// Thin inline-PTX layer over the Hopper (sm_90a) primitives the tensor-core path uses: mbarrier, wgmma (shared-memory
// descriptors, fence / commit / wait), warp-level mma.sync, cp.async and TMA bulk copies.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace egnn {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin (try_wait sleeps in hardware); a bounded variant would hide protocol bugs, an unbounded
// one hangs the GPU on them -- so trap after an absurd number of polls.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) { asm volatile("trap;"); }
  }
}

// The same on a precomputed 32-bit shared-memory address (smem_u32 of a barrier costs an S2UR + ULEA sequence for the
// generic -> shared conversion; hot loops convert once and use these).
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (test_wait never suspends the thread)
__device__ __forceinline__ bool mbar_test_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait_a(bar, parity)) {
    if (++spins > (1u << 28)) { asm volatile("trap;"); }
  }
}

// ------------------------------------------------------------------ proxies / fences
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------ wgmma (one warpgroup of 128 threads)
// Shared-memory matrix descriptor of a K-major operand in the 128-byte-swizzle canonical layout: rows of 128 B
// (64 bf16), groups of 8 rows = 1024 B (`sbo`), the 16-byte chunk index of a row XOR-ed with (row % 8).  Tile base
// 1024-byte aligned; a K=16 step advances the start address by 32 B inside the swizzle atom.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;                      // LBO: unused for swizzled K-major
  d |= (uint64_t)(1024 >> 4) << 32;            // SBO: 8-row group stride
  d |= (uint64_t)1 << 62;                      // layout_type = SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (+)= A * B^T, M=64 N=128 K=16, bf16 operands (both K-major in shared memory), fp32 accumulators in registers.
// Thread t of warp w of the warpgroup holds d[r] = D[16 w + t/4 + 8 ((r >> 1) & 1)][8 (r >> 2) + 2 (t % 4) + (r & 1)].
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,"
      "%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// ------------------------------------------------------------------ warp-level MMA (fused edge kernels)
// D += A * B, M=16 N=8 K=16, bf16 operands and fp32 accumulators in registers (mma.sync fragment layouts: lane
// (lr = l/4, lq = l%4) holds A rows lr / lr+8 and B / D column lr (B) or 2 lq, 2 lq + 1 (D)).
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// One K=16 slab of the fused edge kernels' second GEMM (hidden [32 pairs x 16] . W2 slab^T [16 x 16]) for the 16 pair
// rows of one half of a warp's 32.  The hidden fragment h[0..3] is what the producers pack: h[0] / h[1] = row lr,
// channels 4 lq .. 4 lq + 3, h[2] / h[3] = the same for row lr + 8.  K is a reduction index, so the four channels of a
// lane may stand at mma positions (2 lq, 2 lq + 1 | 2 lq + 8, 2 lq + 9) as long as the B fragment uses the same order:
// then B of lane (lr, lq) for output column n = 8 nt + lr is channels 4 lq .. 4 lq + 3 of W2 row n -- one 8-byte load
// from the core-matrix packing of W2 (slab s at byte 512 s: [kc = k/8][nc = n/8][n % 8][k % 8]).
__device__ __forceinline__ void mma_w2_slab(float (&acc)[2][4], const uint32_t (&h)[4], const unsigned char* w2s, int slab, int lr, int lq) {
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    const uint2 bw = *reinterpret_cast<const uint2*>(w2s + slab * 512 + (lq >> 1) * 256 + nt * 128 + lr * 16 + (lq & 1) * 8);
    mma_16816(acc[nt], h[0], h[2], h[1], h[3], bw.x, bw.y);
  }
}

// ------------------------------------------------------------------ copies into shared memory
// Ampere-style 16-byte async copy with zero-fill when src_bytes == 0 (generic proxy write).
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* gptr, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(gptr), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// TMA bulk copy (no tensor map): `bytes` contiguous bytes global -> shared, completion counted on an
// mbarrier (SASS: UBLKCP).  bytes % 16 == 0, both addresses 16-byte aligned.
__device__ __forceinline__ void tma_bulk_g2s(uint32_t saddr, const void* gptr, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(saddr),
               "l"(gptr), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

template <int V> struct IntC { static constexpr int value = V; };     // compile-time int tag for generic lambdas

// ------------------------------------------------------------------ scalar helpers
// a*b+c for two channels (two FFMAs; kept as one call so the producers read as channel pairs)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// silu(2y) given y = x/2:  x*sigmoid(x) = y + y*tanh(y)
__device__ __forceinline__ float silu_half_arg(float y) { return fmaf(y, tanh_fast(y), y); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// c + (low / high bf16 half of u): a bf16 is the upper half of the fp32 with the same value
__device__ __forceinline__ float add_bf16_lo(uint32_t u, float c) { return __uint_as_float(u << 16) + c; }
__device__ __forceinline__ float add_bf16_hi(uint32_t u, float c) { return __uint_as_float(u & 0xFFFF0000u) + c; }

}  // namespace tc
}  // namespace egnn

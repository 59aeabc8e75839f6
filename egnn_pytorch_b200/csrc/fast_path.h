// bf16 tensor-core ("fast") path: wgmma / mma.sync / TMA kernels for sm_90a (fast_path.cu).
#pragma once
#include "common.cuh"

namespace egnn {
int fast_packed_bytes(const EgnnLayerDesc& d, size_t* out);
int fast_pack_weights(const EgnnLayerDesc& d, const EgnnLayerWeights& w, void* packed, size_t bytes, cudaStream_t st);
int fast_workspace_bytes(const EgnnLayerDesc& d, size_t* out);
int fast_forward(const EgnnLayerDesc& d, const EgnnLayerWeights& w, const void* packed, const EgnnLayerIO& io,
                 const void* box, int pbc, void* ws, size_t ws_bytes, cudaStream_t st);
int debug_gemm_bf16(int M, int N, int K, const void* A, const void* W, const float* bias, float scale, int act,
                    void* out, int out_f32, cudaStream_t st);
}  // namespace egnn

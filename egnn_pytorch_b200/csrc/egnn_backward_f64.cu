// fp64 instantiation of the backward orchestration (its own translation unit: compiles beside the fp32 one).
#include "egnn_backward_impl.cuh"

namespace egnn {
template int simt_backward<double>(const EgnnLayerDesc&, const EgnnLayerWeights&, const void*, const EgnnLayerIO&, const void*, int, const void*,
                                   const EgnnLayerGrads&, double*, void*, size_t, cudaStream_t);
}  // namespace egnn

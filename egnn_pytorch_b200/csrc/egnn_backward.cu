// extern "C" backward entry points (include/egnn_b200.h); the orchestration lives in egnn_backward_impl.cuh.
#include "egnn_backward_impl.cuh"

namespace egnn {

template int simt_backward<float>(const EgnnLayerDesc&, const EgnnLayerWeights&, const void*, const EgnnLayerIO&, const void*, int, const void*,
                                  const EgnnLayerGrads&, double*, void*, size_t, cudaStream_t);
extern template int simt_backward<double>(const EgnnLayerDesc&, const EgnnLayerWeights&, const void*, const EgnnLayerIO&, const void*, int, const void*,
                                          const EgnnLayerGrads&, double*, void*, size_t, cudaStream_t);   // egnn_backward_f64.cu

static int check_grad_ptrs(const EgnnLayerDesc& d, const EgnnLayerGrads* g) {
  if (!g || !g->g_feats_out || !g->g_coors_out || !g->g_feats || !g->g_coors) return EGNN_ERR_NULL;
  const EgnnLayerWeightGrads& w = g->w;
  if (!w.edge_w1 || !w.edge_b1 || !w.edge_w2 || !w.edge_b2) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_SOFT_EDGES) && (!w.gate_w || !w.gate_b)) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_NORM_FEATS) && (d.flags & EGNN_FLAG_UPDATE_FEATS) && (!w.norm_g || !w.norm_b)) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_NORM_COORS) && (d.flags & EGNN_FLAG_UPDATE_COORS) && !w.coors_scale) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_UPDATE_FEATS) && (!w.node_w1 || !w.node_b1 || !w.node_w2 || !w.node_b2)) return EGNN_ERR_NULL;
  if ((d.flags & EGNN_FLAG_UPDATE_COORS) && (!w.coors_w1 || !w.coors_b1 || !w.coors_w2 || !w.coors_b2)) return EGNN_ERR_NULL;
  if (((uintptr_t)g->g_feats | (uintptr_t)g->g_feats_out | (uintptr_t)g->g_edges) & 0xF) return EGNN_ERR_ALIGN;
  return EGNN_OK;
}

}  // namespace egnn

using namespace egnn;

extern "C" int egnn_layer_backward_workspace_bytes(const EgnnLayerDesc* desc, size_t* out_bytes) {
  if (!out_bytes) return EGNN_ERR_NULL;
  EGNN_TRY(validate_desc(desc));
  EGNN_TRY(backward_supported(*desc));
  const Dims s = make_dims(*desc);
  *out_bytes = bwd_ws_layout(s, simt_pack_layout(s), elem_size(desc->dtype), desc->flags).total + 256;
  return EGNN_OK;
}

// box: [B,C] lengths (pbc = PBC_BOX), a [B,C,C] lower-triangular cell (PBC_CELL), or null.  g_lat: null, or the fp64
// gradient with respect to the box / cell (same shape), overwritten.
static int layer_backward(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed, const EgnnLayerIO* io,
                          const void* box, int pbc, const void* fwd_workspace, const EgnnLayerGrads* grads, double* g_lat,
                          void* workspace, size_t workspace_bytes, void* stream) {
  EGNN_TRY(validate_desc(desc));
  if (pbc == PBC_CELL && (desc->C < 2 || desc->C > 3)) return EGNN_ERR_SHAPE;
  EGNN_TRY(backward_supported(*desc));
  if (!io || !packed || !workspace || !fwd_workspace) return EGNN_ERR_NULL;
  EGNN_TRY(check_ptrs(*desc, w, nullptr));
  if (!io->feats || !io->coors) return EGNN_ERR_NULL;
  if (desc->edge_dim > 0 && !io->edges) return EGNN_ERR_NULL;
  if (desc->label_dim > 0 && !io->edge_labels) return EGNN_ERR_NULL;
  if ((desc->flags & EGNN_FLAG_EDGES_PER_SLOT) && !io->nbr_idx) return EGNN_ERR_SHAPE;
  EGNN_TRY(check_grad_ptrs(*desc, grads));
  if (((uintptr_t)workspace | (uintptr_t)fwd_workspace) & 0xFF) return EGNN_ERR_ALIGN;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (desc->dtype == EGNN_DTYPE_F64)
    return simt_backward<double>(*desc, *w, packed, *io, box, pbc, fwd_workspace, *grads, g_lat, workspace, workspace_bytes, st);
  return simt_backward<float>(*desc, *w, packed, *io, box, pbc, fwd_workspace, *grads, g_lat, workspace, workspace_bytes, st);
}

extern "C" int egnn_layer_backward_periodic(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                            const EgnnLayerIO* io, const void* box, const void* fwd_workspace,
                                            const EgnnLayerGrads* grads, void* workspace, size_t workspace_bytes, void* stream) {
  return layer_backward(desc, w, packed, io, box, PBC_BOX, fwd_workspace, grads, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int egnn_layer_backward_periodic_lattice(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                                    const EgnnLayerIO* io, const void* box, const void* fwd_workspace,
                                                    const EgnnLayerGrads* grads, double* g_box, void* workspace,
                                                    size_t workspace_bytes, void* stream) {
  if (!box || !g_box) return EGNN_ERR_NULL;
  return layer_backward(desc, w, packed, io, box, PBC_BOX, fwd_workspace, grads, g_box, workspace, workspace_bytes, stream);
}

extern "C" int egnn_layer_backward_triclinic(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                             const EgnnLayerIO* io, const void* cell, const void* fwd_workspace,
                                             const EgnnLayerGrads* grads, void* workspace, size_t workspace_bytes,
                                             void* stream) {
  if (!cell) return EGNN_ERR_NULL;
  return layer_backward(desc, w, packed, io, cell, PBC_CELL, fwd_workspace, grads, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int egnn_layer_backward_triclinic_lattice(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                                     const EgnnLayerIO* io, const void* cell, const void* fwd_workspace,
                                                     const EgnnLayerGrads* grads, double* g_cell, void* workspace,
                                                     size_t workspace_bytes, void* stream) {
  if (!cell || !g_cell) return EGNN_ERR_NULL;
  return layer_backward(desc, w, packed, io, cell, PBC_CELL, fwd_workspace, grads, g_cell, workspace, workspace_bytes, stream);
}

extern "C" int egnn_layer_backward(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                   const EgnnLayerIO* io, const void* fwd_workspace, const EgnnLayerGrads* grads,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  return egnn_layer_backward_periodic(desc, w, packed, io, nullptr, fwd_workspace, grads, workspace, workspace_bytes, stream);
}

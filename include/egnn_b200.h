/*
 * egnn_b200.h -- C ABI of libegnn_b200.so, the H100 (sm_90a) implementation of the
 * E(n)-equivariant message-passing layer of lucidrains/egnn-pytorch.
 *
 * The reference has no FFI: its boundary is the Python nn.Module API
 * (reference egnn_pytorch/__init__.py:1, EGNN.forward egnn_pytorch/egnn_pytorch.py:224-341,
 * EGNN_Network.forward :390-454).  This header is the boundary a binding for that path
 * would target; `egnn_pytorch_b200/egnn.py` is such a binding (ctypes), keeping the
 * reference's module names, constructor arguments, forward signatures and state-dict keys.
 *
 * Conventions
 *  - plain C, no CUDA or torch types: device pointers are `void*` / `const void*`,
 *    the stream is the `cudaStream_t` handle passed as `void*` (NULL = default stream);
 *  - the library BORROWS every pointer for the duration of the call, allocates nothing that
 *    outlives the call and never synchronises the stream (HOST-buffer entry excepted);
 *  - every entry returns 0 on success or a negative EGNN_ERR_* code and never throws;
 *  - all tensors are contiguous, row-major, in the layouts written next to each field;
 *  - re-entrant across streams and devices; the only mutable global state is a mutex-guarded, write-once per-device
 *    cache of kernel attributes / SM counts and the opt-in profiler below.
 */
#ifndef EGNN_B200_H_
#define EGNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EGNN_ABI_VERSION 4   /* 2: EgnnLayerIO grew nbr_idx + pre2_out; backward entry points added
                                3: peer-memory all-gather communicator (egnn_comm_*), egnn_global_attn_*
                                4: EGNN_FLAG_EDGES_PER_SLOT (io.edges / g_edges per neighbour slot);
                                   EGNN_FLAG_ROW_PARTIAL_GRADS (backward of a row block) added later as one more flag bit,
                                   the descriptor unchanged.  A version-4 library that predates it ignores the bit, and its
                                   backward preflight (egnn_layer_backward_workspace_bytes, which a training caller runs
                                   before the forward) still rejects the row range with EGNN_ERR_UNSUPPORTED: a mismatch
                                   fails loudly before anything is written into block-sized buffers */

/* ---- error codes ------------------------------------------------------------------- */
#define EGNN_OK                 0
#define EGNN_ERR_NULL          -1   /* required pointer is NULL                           */
#define EGNN_ERR_SHAPE         -2   /* inconsistent / out-of-range sizes                  */
#define EGNN_ERR_UNSUPPORTED   -3   /* option combination this build has no kernel for    */
#define EGNN_ERR_ALIGN         -4   /* pointer not aligned as documented (16 bytes)       */
#define EGNN_ERR_WORKSPACE     -5   /* workspace / packed buffer too small                */
#define EGNN_ERR_ABI           -6   /* desc.abi_version != EGNN_ABI_VERSION               */
#define EGNN_ERR_CUDA       -1000   /* -(1000 + cudaError_t) for CUDA runtime failures    */

/* ---- element types of feats / edges / weights / outputs ---------------------------- */
#define EGNN_DTYPE_F32   0   /* SIMT fp32 kernels ("accurate" path)                       */
#define EGNN_DTYPE_F64   1   /* SIMT fp64 kernels (the reference's tests run in fp64)     */
#define EGNN_DTYPE_BF16  2   /* bf16 tensor-core kernels (wgmma / mma.sync), fp32 accum.   */

/* ---- flags (EgnnLayerDesc.flags) ---------------------------------------------------- */
#define EGNN_FLAG_NORM_FEATS    (1u << 0)   /* node_norm = LayerNorm  (egnn_pytorch.py:191)   */
#define EGNN_FLAG_NORM_COORS    (1u << 1)   /* coors_norm = CoorsNorm (:192, :67-77)          */
#define EGNN_FLAG_UPDATE_FEATS  (1u << 2)   /* node_mlp present       (:196-201)              */
#define EGNN_FLAG_UPDATE_COORS  (1u << 3)   /* coors_mlp present      (:203-208)              */
#define EGNN_FLAG_SOFT_EDGES    (1u << 4)   /* edge_gate present      (:186-189)              */
#define EGNN_FLAG_POOL_MEAN     (1u << 5)   /* m_pool_method == 'mean' (:325-330)             */
#define EGNN_FLAG_CLAMP         (1u << 6)   /* coor_weights_clamp_value is set (:311-313)     */
#define EGNN_FLAG_ONLY_SPARSE   (1u << 7)   /* only_sparse_neighbors: valid_radius := 0 (:250);
                                               the caller passes k = max adjacency row sum   */
#define EGNN_FLAG_ADJ_BATCHED   (1u << 8)   /* io.adj is [B,N,N] instead of [N,N] (:245)      */
#define EGNN_FLAG_EDGES_PER_SLOT (1u << 9)  /* io.edges / grads.g_edges are [B,N,k,edge_dim], aligned with the caller's
                                               io.nbr_idx: slot s of row i holds edge nbr_idx[b,i,s] -> i.  Needs
                                               k > 0 and edge_dim > 0 (else EGNN_ERR_SHAPE) and io.nbr_idx != NULL
                                               (EGNN_ERR_SHAPE from egnn_layer_forward / egnn_layer_backward) */
#define EGNN_FLAG_ROW_PARTIAL_GRADS (1u << 10) /* training of a row block [row_begin, row_end) (row-sharded graphs): pass the
                                               same desc to egnn_layer_forward and egnn_layer_backward.  io.pre2_out and the
                                               backward's per-pair buffers are sized by the block, [B, R, J, *] with
                                               R = row_end - row_begin; egnn_layer_backward returns the gradient of
                                               sum_{b, i in block} <g_out[b,i], out[b,i]>.  See EgnnLayerGrads */
#define EGNN_FLAG_CELL_SELECT_WIDE (1u << 11) /* lets a layer with 32 < k <= 256 select its lists on the cell grid
                                               (egnn_radius_select_wide) when it is otherwise eligible (C <= 3, a finite
                                               valid_radius, no adjacency or per-slot edges; DESIGN.md section 5).  Such a
                                               descriptor's workspace ends in the cell grid's scratch.  Without the flag a
                                               layer with k > 32 ranks all pairs, and its workspace is unchanged */
#define EGNN_FLAG_KNN_GRID (1u << 12)         /* lets a layer select its k nearest neighbours on the kNN cell grid
                                               (egnn_knn_grid_select) when the radius grid does not run and the layer
                                               is eligible: C <= 3, 1 <= k <= 32 (<= 256 with EGNN_FLAG_CELL_SELECT_WIDE),
                                               no adjacency, only_sparse, caller lists or per-slot edges, and N at least
                                               a size threshold (EGNN_B200_KNN_GRID_MIN_N overrides it per call).  The
                                               lists equal the all-pairs select's.  Such a descriptor's workspace ends in
                                               the kNN grid's scratch; without the flag nothing changes */

/*
 * Static description of one layer call.  E = 2*dim + 2*fourier + 1 + edge_dim + label_dim
 * is the reference's edge_input_dim (egnn_pytorch.py:175); H = 2*E.
 */
typedef struct EgnnLayerDesc {
  int32_t  abi_version;   /* EGNN_ABI_VERSION                                             */
  int32_t  dtype;         /* EGNN_DTYPE_*                                                 */
  int32_t  B, N;          /* graphs, nodes per graph                                      */
  int32_t  C;             /* coordinate dimension, 1..8 (tests/test_equivariance.py:40 uses 5) */
  int32_t  dim;           /* node feature width                                           */
  int32_t  edge_dim;      /* continuous edge channels read from io.edges (0 = none)       */
  int32_t  label_dim;     /* columns of edge_mlp.0.weight fed by the label embedding (adj_dim,
                             egnn_pytorch.py:430-432), 0 = none                           */
  int32_t  num_labels;    /* rows of weights.label_emb                                    */
  int32_t  m_dim;         /* message width (default 16), <= 32                            */
  int32_t  fourier;       /* fourier_features                                             */
  int32_t  k;             /* 0 = dense all-pairs; >0 = neighbours per node, i.e. the reference's
                             use_nearest branch (:237-268) with num_nearest = k           */
  uint32_t flags;         /* EGNN_FLAG_*                                                  */
  int32_t  row_begin;     /* evaluate i-rows [row_begin, row_end) only (row-sharded multi-GPU); */
  int32_t  row_end;       /*   0,0 = all rows.  Outputs keep their full [B,N,*] layout.   */
  int32_t  reserved;      /* must be 0                                                    */
  double   valid_radius;  /* used only when k>0 AND io.mask != NULL (:260, :296); +inf ok */
  double   clamp;         /* coor_weights_clamp_value when EGNN_FLAG_CLAMP                */
  double   dropout_p;     /* training-mode dropout probability of edge_mlp / node_mlp / coors_mlp (egnn_pytorch.py:176-208);
                             0 = off (eval mode).  fp32 / fp64 kernels only.                */
  uint64_t dropout_seed;  /* masks are regenerated from (seed, element index) in forward AND backward: pass the SAME
                             desc to egnn_layer_backward; draw a fresh seed per training step */
} EgnnLayerDesc;

/*
 * Device pointers to the layer's parameters, each exactly as nn.Linear / nn.LayerNorm stores it
 * (row-major [out, in]) under the state-dict key named on the right.  Element type = desc.dtype.
 * Pointers for modules the flags disable may be NULL.
 */
typedef struct EgnnLayerWeights {
  const void* edge_w1;    /* [H, E]      edge_mlp.0.weight   */
  const void* edge_b1;    /* [H]         edge_mlp.0.bias     */
  const void* edge_w2;    /* [m, H]      edge_mlp.3.weight   */
  const void* edge_b2;    /* [m]         edge_mlp.3.bias     */
  const void* gate_w;     /* [1, m]      edge_gate.0.weight  */
  const void* gate_b;     /* [1]         edge_gate.0.bias    */
  const void* norm_g;     /* [dim]       node_norm.weight    */
  const void* norm_b;     /* [dim]       node_norm.bias      */
  const void* coors_scale;/* [1]         coors_norm.scale    */
  const void* node_w1;    /* [2dim, dim+m]  node_mlp.0.weight */
  const void* node_b1;    /* [2dim]      node_mlp.0.bias     */
  const void* node_w2;    /* [dim, 2dim] node_mlp.3.weight   */
  const void* node_b2;    /* [dim]       node_mlp.3.bias     */
  const void* coors_w1;   /* [4m, m]     coors_mlp.0.weight  */
  const void* coors_b1;   /* [4m]        coors_mlp.0.bias    */
  const void* coors_w2;   /* [1, 4m]     coors_mlp.3.weight  */
  const void* coors_b2;   /* [1]         coors_mlp.3.bias    */
  const void* label_emb;  /* [num_labels, label_dim]  EGNN_Network.adj_emb.weight (or NULL) */
} EgnnLayerWeights;

/*
 * Per-call tensors (device memory).  feats/edges/feats_out have element type desc.dtype;
 * coors/coors_out are float64 when desc.dtype == F64 and float32 otherwise.
 */
typedef struct EgnnLayerIO {
  const void*    feats;      /* [B, N, dim]                                               */
  const void*    coors;      /* [B, N, C]                                                 */
  const void*    edges;      /* [B, N, N, edge_dim], or [B, N, k, edge_dim] per neighbour slot under
                                EGNN_FLAG_EDGES_PER_SLOT; NULL when edge_dim == 0                */
  const uint8_t* edge_labels;/* [B, N, N] label index per pair, or NULL when label_dim == 0 */
  const uint8_t* mask;       /* [B, N] 0/1, or NULL (= the reference's mask=None)         */
  const uint8_t* adj;        /* [N, N] or [B, N, N] 0/1 (EGNN_FLAG_ADJ_BATCHED), or NULL;
                                only read when k > 0                                      */
  void*          feats_out;  /* [B, N, dim]                                               */
  void*          coors_out;  /* [B, N, C]                                                 */
  const int32_t* nbr_idx;    /* optional, k > 0 only: caller-supplied neighbour lists [B, N, k] (edge-list
                                mode, SURVEY.md section 8(f) rank 3): the distance/top-k pass is skipped.  An entry
                                < 0 is an empty slot and never contributes.  NULL = select as the reference does. */
  void*          pre2_out;   /* optional, fp32/fp64 training only: [B, N, J, MP] with J = N (dense) or k (neighbour lists)
                                and MP = 16 when m_dim <= 16, else 32.  egnn_layer_forward stores the per-pair
                                pre-activation of edge_mlp's second SiLU there; egnn_layer_backward, given the same
                                pointer, skips recomputing it -- a speed / memory trade (64 B per pair in fp32).
                                NULL = nothing stored, backward recomputes.  Under EGNN_FLAG_ROW_PARTIAL_GRADS
                                [B, R, J, MP]: the pairs of rows [row_begin, row_end) only, row i at i - row_begin. */
} EgnnLayerIO;

int         egnn_abi_version(void);
const char* egnn_strerror(int code);

/* Bytes of the packed-parameter buffer for `desc` (depends on dtype and sizes only). */
int egnn_layer_packed_bytes(const EgnnLayerDesc* desc, size_t* out_bytes);

/* Re-layout the parameters for the kernels (split W1 into per-node and per-pair parts,
 * transpose W2, fold the label embedding into a [num_labels, H] table, bf16 copies for the
 * tensor-core path).  Enqueued on `stream`; call again whenever a parameter changes. */
int egnn_layer_pack_weights(const EgnnLayerDesc* desc, const EgnnLayerWeights* w,
                            void* packed, size_t packed_bytes, void* stream);

/* Bytes of scratch `egnn_layer_forward` needs for `desc` (per-node tables, neighbour lists). */
int egnn_layer_workspace_bytes(const EgnnLayerDesc* desc, size_t* out_bytes);

/* One EGNN layer forward == reference EGNN.forward (egnn_pytorch.py:224-341), enqueued on
 * `stream`.  `packed` comes from egnn_layer_pack_weights with an identical desc (B, N, k,
 * flags and the row range may differ).  `workspace` must be 256-byte aligned. */
int egnn_layer_forward(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                       const EgnnLayerIO* io, void* workspace, size_t workspace_bytes,
                       void* stream);

/* Periodic boundaries: egnn_layer_forward with every pair geometry x_i - x_j replaced by its minimum image
 *   rel_c - L_c * rint(rel_c / L_c)   (rounding half to even; 1/L_c is formed once per row or CTA)
 * on each axis c with a finite box length L_c > 0; an axis with L_c = 0 or +inf is not periodic.  The distance, its
 * fourier features, the neighbour ranking (valid_radius, adjacency ranks unchanged), CoorsNorm and the coordinate update
 * x_i + sum_j w_ij rel_ij all use the wrapped rel; the output coordinates are not wrapped back into the box.
 * `box`: device [B, C] in the coordinates' type (float64 for EGNN_DTYPE_F64, else float32), lengths >= 0 or +inf;
 * NULL = egnn_layer_forward.  Orthorhombic boxes only, one image per neighbour. */
int egnn_layer_forward_periodic(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                const EgnnLayerIO* io, const void* box, void* workspace, size_t workspace_bytes,
                                void* stream);

/* Triclinic cells: egnn_layer_forward_periodic with a lattice in place of the box.  `cell`: device [B, C, C], row-major,
 * in the coordinates' type, C in {2, 3} (EGNN_ERR_SHAPE otherwise); row k is lattice vector a_k and the cell is lower-
 * triangular (cell[k][d] == 0 for d > k).  A diagonal entry of 0 or +inf marks axis k aperiodic; its row and column
 * must then be zero off the diagonal.  Every pair vector is wrapped sequentially from the last axis to the first: for
 * c = C-1 .. 0 with L_c = cell[c][c] periodic, n = rint(r_c * (1/L_c)), then r_d -= cell[c][d] * n (one fma) for every
 * d <= c.  After the wrap |r_c| <= L_c / 2 on every periodic axis: the result lies in the centred box of the diagonal
 * entries, a fundamental domain of the lattice, so it is the minimum image whenever the minimum image is shorter than
 * min_c L_c / 2; pairs farther apart get that centred-box image, one image per neighbour.  A diagonal cell gives the
 * outputs of egnn_layer_forward_periodic with its diagonal as the box, bit for bit.  The values are not validated here.
 * Workspace and packed sizes are those of egnn_layer_forward. */
int egnn_layer_forward_triclinic(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                 const EgnnLayerIO* io, const void* cell, void* workspace, size_t workspace_bytes,
                                 void* stream);

/* Same call with HOST buffers for io.* (pinned or pageable): allocates device staging,
 * copies in, runs, copies feats_out / coors_out back and synchronises.  Parameters (`w`,
 * `packed`) stay device-resident.  This is the end-to-end entry `bench.py` times as `e2e`. */
int egnn_layer_forward_host(const EgnnLayerDesc* desc, const EgnnLayerWeights* w,
                            const void* packed, const EgnnLayerIO* host_io, void* stream);

/*
 * Backward of one layer (SURVEY.md section 8(f) rank 1): what autograd computes through the reference's
 * EGNN.forward (egnn_pytorch.py:224-341).  fp32 / fp64 kernels only (EGNN_ERR_UNSUPPORTED for bf16 and for a row
 * range without EGNN_FLAG_ROW_PARTIAL_GRADS).  The edge step is recomputed pair by pair, so the only saved state is
 * the forward WORKSPACE: `fwd_workspace` must be the buffer egnn_layer_forward ran on with the same desc / io,
 * unmodified since.  Gradient buffers are OVERWRITTEN (not accumulated into).  Neighbour selection contributes no
 * gradient.
 *
 * Row blocks (EGNN_FLAG_ROW_PARTIAL_GRADS with a row range): the gradient of sum_{b, i in [row_begin, row_end)}
 * <g_out[b,i], out[b,i]>.  Only the block's rows of g_feats_out / g_coors_out are read.  g_feats, g_coors, g_edges and
 * every weight gradient keep their full shapes and hold this block's contribution: the block's own rows (residual,
 * node update, dL/dA_i), the neighbour-side terms of every row j (dL/dB_j, dL/dx_j, edges), 0 where there are none.
 * Summed over the blocks of a partition of the rows they give the gradient of the whole layer.  Dropout masks are keyed
 * on global indices, so the blocks see the masks of the whole-graph call with the same seed.
 */
typedef struct EgnnLayerWeightGrads {   /* one buffer per EgnnLayerWeights field, same shape and dtype; NULL for
                                           modules the flags disable */
  void* edge_w1; void* edge_b1; void* edge_w2; void* edge_b2; void* gate_w; void* gate_b;
  void* norm_g; void* norm_b; void* coors_scale;
  void* node_w1; void* node_b1; void* node_w2; void* node_b2;
  void* coors_w1; void* coors_b1; void* coors_w2; void* coors_b2; void* label_emb;
} EgnnLayerWeightGrads;

typedef struct EgnnLayerGrads {
  const void* g_feats_out;   /* [B, N, dim]  dL/d feats_out (input)                         */
  const void* g_coors_out;   /* [B, N, C]    dL/d coors_out (input)                         */
  void*       g_feats;       /* [B, N, dim]  dL/d feats                                     */
  void*       g_coors;       /* [B, N, C]    dL/d coors                                     */
  void*       g_edges;       /* [B, N, N, edge_dim] dL/d edges, or NULL (not wanted / edge_dim == 0).
                                Under EGNN_FLAG_EDGES_PER_SLOT [B, N, k, edge_dim]: one plain store per slot, no
                                atomics across slots; empty (-1) slots get 0                     */
  EgnnLayerWeightGrads w;
} EgnnLayerGrads;

int egnn_layer_backward_workspace_bytes(const EgnnLayerDesc* desc, size_t* out_bytes);
int egnn_layer_backward(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                        const EgnnLayerIO* io, const void* fwd_workspace, const EgnnLayerGrads* grads,
                        void* workspace, size_t workspace_bytes, void* stream);
/* Backward of egnn_layer_forward_periodic: pass the SAME `box` as the forward (NULL = egnn_layer_backward).  The wrap's
 * derivative with respect to the coordinates is the identity; egnn_layer_backward_periodic_lattice adds the gradient
 * with respect to the box. */
int egnn_layer_backward_periodic(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                 const EgnnLayerIO* io, const void* box, const void* fwd_workspace,
                                 const EgnnLayerGrads* grads, void* workspace, size_t workspace_bytes, void* stream);
/* Backward of egnn_layer_forward_triclinic: pass the SAME `cell` as the forward.  egnn_layer_backward_triclinic_lattice
 * adds the gradient with respect to the cell. */
int egnn_layer_backward_triclinic(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                  const EgnnLayerIO* io, const void* cell, const void* fwd_workspace,
                                  const EgnnLayerGrads* grads, void* workspace, size_t workspace_bytes, void* stream);
/* Lattice gradients (stress / virial): egnn_layer_backward_periodic / _triclinic, returning every gradient they return,
 * plus the gradient of the loss with respect to the box or the cell.  The wrap is rel = (x_i - x_j) - sum_c n_c a_c with
 * integer image counts n (piecewise constant), so with gr = dL/d rel of a pair
 *   g_box  [B, C]    (float64): g_box[b][c]     = - sum_pairs n_c gr_c;
 *   g_cell [B, C, C] (float64): g_cell[b][c][d] = - sum_pairs n_c gr_d for d <= c, 0 above the diagonal;
 * 0 on aperiodic axes and rows.  Neighbour selection contributes nothing.  The buffer is overwritten (zeroed on the
 * stream) and accumulated in float64 whatever the layer's type, with atomics: reproducible to fp64 rounding.  A row
 * block (EGNN_FLAG_ROW_PARTIAL_GRADS) returns its share, so the shares of a partition of the rows sum to the whole.
 * A NULL box / cell or gradient: EGNN_ERR_NULL; C outside {2, 3} for a cell: EGNN_ERR_SHAPE.  Same workspace. */
int egnn_layer_backward_periodic_lattice(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                         const EgnnLayerIO* io, const void* box, const void* fwd_workspace,
                                         const EgnnLayerGrads* grads, double* g_box, void* workspace,
                                         size_t workspace_bytes, void* stream);
int egnn_layer_backward_triclinic_lattice(const EgnnLayerDesc* desc, const EgnnLayerWeights* w, const void* packed,
                                          const EgnnLayerIO* io, const void* cell, const void* fwd_workspace,
                                          const EgnnLayerGrads* grads, double* g_cell, void* workspace,
                                          size_t workspace_bytes, void* stream);

/* Neighbour selection alone == ranking + topk of egnn_pytorch.py:237-260: for every node the k
 * lowest-ranked nodes (rank = squared distance; 1e5 if either end is masked out; -1 self and 0
 * adjacent when `adj` is given), ascending, ties to the lowest index.
 * coors [B,N,C] (float32, or float64 when dtype == EGNN_DTYPE_F64); mask/adj as in EgnnLayerIO;
 * out_idx int32 [B,N,k]; out_ok uint8 [B,N,k] = (rank <= valid_radius), may be NULL. */
int egnn_knn_select(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k,
                    const void* coors, const uint8_t* mask, const uint8_t* adj, int32_t adj_batched,
                    double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* stream);

/* Neighbour lists from an adjacency alone: slot 0 = the node itself, then its adjacent nodes in ascending index order,
 * truncated at k -- exactly the slots of egnn_knn_select whose rank is <= 0 (egnn_pytorch.py:255-256), i.e. every slot that
 * survives `only_sparse_neighbors` with a node mask (valid_radius = 0, :250, :296).  They do not depend on the coordinates,
 * so EGNN_Network builds them once per adjacency and hands them to every layer (EgnnLayerIO.nbr_idx).
 * adj [N,N] or [B,N,N] 0/1 bytes; out_idx int32 [B,N,k]; out_ok uint8 [B,N,k] or NULL.  Unused slots: the node itself with
 * ok = 0, or -1 when out_ok is NULL. */
int egnn_adj_neighbors(int32_t B, int32_t N, int32_t k, const uint8_t* adj, int32_t adj_batched, int32_t* out_idx,
                       uint8_t* out_ok, void* stream);

/* Radius graph from a cell grid, O(N) instead of egnn_knn_select's O(N^2): for every node the k lowest-ranked nodes
 * with rank <= r2, ascending, ties to the lowest index -- exactly the ok = 1 slots of egnn_knn_select with the same
 * coordinates, mask and valid_radius = r2 (rank = squared distance computed in the coordinates' type; minimum image
 * under `box`).  A padded node (mask 0) or one with a non-finite coordinate is never a neighbour, and its own row is
 * empty.  egnn_layer_forward runs the same search for an eligible layer (k <= 32, or k <= 256 under
 * EGNN_FLAG_CELL_SELECT_WIDE; C <= 3, a mask, a finite valid_radius, no adjacency; DESIGN.md section 5) once N
 * reaches a size threshold (EGNN_B200_CELL_SELECT_MIN_N).
 * coors [B,N,C] (float32, or float64 when dtype == EGNN_DTYPE_F64); mask [B,N] 0/1 or NULL (all valid); box [B,C] in
 * the coordinates' type or NULL, as egnn_layer_forward_periodic takes it; r2 > 0 (EGNN_ERR_SHAPE otherwise), a squared
 * distance, compared as (float)r2 for float32 coordinates.  out_idx int32 [B,N,k]: the kept neighbours, then -1 in every
 * remaining slot (the edge-list convention of EgnnLayerIO.nbr_idx); out_count int32 [B,N] or NULL: the number of nodes
 * with rank <= r2 before the truncation at k (the node itself included).  k <= 32 and C <= 3, else EGNN_ERR_UNSUPPORTED.
 * workspace: egnn_radius_select_workspace_bytes(B, N, C, k) bytes (O(B N), enough for either coordinate type),
 * 256-byte aligned.  Enqueued on `stream`, no host synchronisation (CUDA-graph capturable). */
int egnn_radius_select_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes);
int egnn_radius_select(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors, const uint8_t* mask,
                       const void* box, double r2, int32_t* out_idx, int32_t* out_count, void* workspace,
                       size_t workspace_bytes, void* stream);
/* egnn_radius_select under a triclinic cell [B, C, C] (as egnn_layer_forward_triclinic takes it; C in {2, 3}, else
 * EGNN_ERR_SHAPE): the ok = 1 slots of the all-pairs select with the rank of the wrapped pair vector.  Periodic axes
 * are binned in fractional coordinates.  Same workspace. */
int egnn_radius_select_triclinic(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                 const uint8_t* mask, const void* cell, double r2, int32_t* out_idx, int32_t* out_count,
                                 void* workspace, size_t workspace_bytes, void* stream);
/* egnn_radius_select / egnn_radius_select_triclinic / their workspace size for lists of 1 <= k <= min(256, N)
 * (k > 256: EGNN_ERR_UNSUPPORTED); the same arguments, checks, error codes and workspace.  For k <= 32 the output is
 * exactly that of the k <= 32 entries; longer lists are kept in shared memory instead of a warp's lanes, with the same
 * result: the ok = 1 slots of egnn_knn_select, independent of the order the grid was filled in. */
int egnn_radius_select_wide_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes);
int egnn_radius_select_wide(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                            const uint8_t* mask, const void* box, double r2, int32_t* out_idx, int32_t* out_count,
                            void* workspace, size_t workspace_bytes, void* stream);
int egnn_radius_select_wide_triclinic(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                      const uint8_t* mask, const void* cell, double r2, int32_t* out_idx,
                                      int32_t* out_count, void* workspace, size_t workspace_bytes, void* stream);

/* k-nearest-neighbour lists from a cell grid, O(N) per graph instead of egnn_knn_select's O(N^2): out_idx and out_ok
 * equal egnn_knn_select's with the same coordinates, mask and valid_radius (no adjacency) bit for bit -- the same rank
 * (squared distance in the coordinates' type, minimum image under `box`), ascending, ties to the lowest index, 1e5 to
 * and from padded nodes, NaN ranks last, ok = (rank <= valid_radius).  Each graph sizes its grid on the device from the
 * extent of its nodes; rows the grid cannot decide (non-finite coordinates, fewer than k valid nodes, a k-th rank at
 * the 1e5 of padded pairs, very uneven clouds) are ranked against every node of their graph (DESIGN.md section 5).
 * coors [B,N,C] (float32, or float64 when dtype == EGNN_DTYPE_F64); mask [B,N] 0/1 or NULL; box [B,C] or NULL as
 * egnn_radius_select takes it; out_idx int32 [B,N,k]; out_ok uint8 [B,N,k] or NULL.  1 <= k <= min(256, N) and C <= 3
 * (k > 256 or C > 3: EGNN_ERR_UNSUPPORTED).  workspace: egnn_knn_grid_select_workspace_bytes(B, N, C, k) bytes (O(B N),
 * enough for either coordinate type), 256-byte aligned.  Enqueued on `stream`, no host synchronisation. */
int egnn_knn_grid_select_workspace_bytes(int32_t B, int32_t N, int32_t C, int32_t k, size_t* out_bytes);
int egnn_knn_grid_select(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                         const uint8_t* mask, const void* box, double valid_radius, int32_t* out_idx, uint8_t* out_ok,
                         void* workspace, size_t workspace_bytes, void* stream);
/* egnn_knn_grid_select under a triclinic cell [B, C, C] (C in {2, 3}, else EGNN_ERR_SHAPE), as egnn_radius_select_triclinic
 * takes it: egnn_knn_select's lists with the rank of the wrapped pair vector.  Same workspace. */
int egnn_knn_grid_select_triclinic(int32_t dtype, int32_t B, int32_t N, int32_t C, int32_t k, const void* coors,
                                   const uint8_t* mask, const void* cell, double valid_radius, int32_t* out_idx,
                                   uint8_t* out_ok, void* workspace, size_t workspace_bytes, void* stream);

/* k-nearest-neighbour lists of a packed batch: G graphs of n_g = ptr[g+1] - ptr[g] nodes laid end to end on one node
 * axis of T nodes (PyTorch Geometric's `ptr`).  Every node is ranked against the nodes of its own graph only, in
 * O(sum_g n_g^2): out_idx and out_ok of node i of graph g equal egnn_knn_select's for that graph alone (B = 1, N = n_g,
 * the same k, mask, valid_radius and lattice) bit for bit, with indices into the node axis (local index + ptr[g]).
 * Slots past n_g (n_g < k) hold -1 with ok = 0; an empty graph writes nothing.
 * ptr int32 [G+1] (device memory, read on the device only, so the call can be captured in a CUDA graph; the graph
 * bounds are clamped to [0, T], and callers pass ptr[0] = 0, non-decreasing, ptr[G] = T); coors [T,C] (float32, or
 * float64 when dtype == EGNN_DTYPE_F64), 1 <= C <= 8; mask [T] 0/1 or NULL; box [C] shared by every graph or NULL;
 * out_idx int32 [T,k]; out_ok uint8 [T,k] or NULL.  1 <= k <= 256 (k > 256: EGNN_ERR_UNSUPPORTED), T <= 2^30.
 * workspace: egnn_knn_select_packed_workspace_bytes(G, T, C, k) bytes (O(G)), 256-byte aligned.  Enqueued on
 * `stream`, no host synchronisation. */
int egnn_knn_select_packed_workspace_bytes(int32_t G, int32_t T, int32_t C, int32_t k, size_t* out_bytes);
int egnn_knn_select_packed(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, const int32_t* ptr,
                           const void* coors, const uint8_t* mask, const void* box, double valid_radius, int32_t* out_idx,
                           uint8_t* out_ok, void* workspace, size_t workspace_bytes, void* stream);
/* egnn_knn_select_packed under a triclinic cell [C, C] shared by every graph (C in {2, 3}, else EGNN_ERR_SHAPE), as
 * egnn_knn_grid_select_triclinic takes one graph's cell.  Same workspace. */
int egnn_knn_select_packed_triclinic(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, const int32_t* ptr,
                                     const void* coors, const uint8_t* mask, const void* cell, double valid_radius,
                                     int32_t* out_idx, uint8_t* out_ok, void* workspace, size_t workspace_bytes,
                                     void* stream);

/* egnn_knn_select_packed with the graphs large enough on a cell grid, as each graph's unpacked call would run: the
 * arguments of egnn_knn_select_packed(_triclinic) plus max_n, the node count of the largest graph (it only decides
 * whether the grid is launched at all).  Graph g goes on the grid when C <= 3, n_g >= k and n_g reaches the threshold
 * read at this call; every other graph (and every graph when ptr is not non-decreasing within [0, T]) on the segmented
 * all-pairs select.  When max_n is below the threshold, the call issues exactly egnn_knn_select_packed's launches.
 * T <= 2^29 - 1 (4 T bucket offsets stay an int, else EGNN_ERR_SHAPE).  workspace: the entry's _workspace_bytes(G, T,
 * C, k) bytes (O(G + T), a function of G, T and C).  No host synchronisation.
 *   egnn_knn_grid_select_packed: the kNN grid from EGNN_B200_KNN_GRID_MIN_N nodes (8192); out_idx and out_ok equal
 *     egnn_knn_select_packed's bit for bit.
 *   egnn_radius_select_packed: the radius grid from EGNN_B200_CELL_SELECT_MIN_N nodes (4096), when 0 < valid_radius
 *     < 1e5 in the coordinates' type (the squared cutoff); out_ok (required) equals egnn_knn_select_packed's and
 *     out_idx equals its idx in every ok = 1 slot (the kept slots; the rest are unspecified). */
int egnn_radius_select_packed_workspace_bytes(int32_t G, int32_t T, int32_t C, int32_t k, size_t* out_bytes);
int egnn_radius_select_packed(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                              const int32_t* ptr, const void* coors, const uint8_t* mask, const void* box,
                              double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                              size_t workspace_bytes, void* stream);
int egnn_radius_select_packed_triclinic(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                                        const int32_t* ptr, const void* coors, const uint8_t* mask, const void* cell,
                                        double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                        size_t workspace_bytes, void* stream);
int egnn_knn_grid_select_packed_workspace_bytes(int32_t G, int32_t T, int32_t C, int32_t k, size_t* out_bytes);
int egnn_knn_grid_select_packed(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                                const int32_t* ptr, const void* coors, const uint8_t* mask, const void* box,
                                double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                size_t workspace_bytes, void* stream);
int egnn_knn_grid_select_packed_triclinic(int32_t dtype, int32_t G, int32_t T, int32_t C, int32_t k, int32_t max_n,
                                          const int32_t* ptr, const void* coors, const uint8_t* mask, const void* cell,
                                          double valid_radius, int32_t* out_idx, uint8_t* out_ok, void* workspace,
                                          size_t workspace_bytes, void* stream);

/* N-th degree adjacency of EGNN_Network (egnn_pytorch.py:414-428) without the dense A@A:
 * adj_in [N,N] or [B,N,N] 0/1; writes the expanded adjacency adj_out [B,N,N] 0/1, the degree
 * labels labels_out [B,N,N] (0 = not connected, d = first reached in round d) and
 * max_row_sum[0] = max over rows of sum_j adj_out (the reference's `num_nearest` under
 * only_sparse_neighbors, :249).  workspace: egnn_adj_workspace_bytes(B, N). */
int egnn_adj_workspace_bytes(int32_t B, int32_t N, size_t* out_bytes);
int egnn_adj_expand(int32_t B, int32_t N, int32_t num_degrees, const uint8_t* adj_in,
                    int32_t adj_batched, uint8_t* adj_out, uint8_t* labels_out,
                    int32_t* max_row_sum, void* workspace, size_t workspace_bytes, void* stream);

/* Node embedding of EGNN_Network (egnn_pytorch.py:401-408) in one launch: out[b,n,:] = token_emb[tokens[b,n],:] +
 * pos_emb[n,:] (pos_emb may be NULL).  Tables and output have element type `dtype`; tokens are int64 [B,N]. */
int egnn_embed_nodes(int32_t dtype, int32_t B, int32_t N, int32_t dim, int32_t num_tokens, const int64_t* tokens,
                     const void* token_emb, const void* pos_emb, void* out, void* stream);

/* The wgmma GEMM the bf16 path uses for its per-node contractions, exposed for unit tests:
 * out[M,N] = act(scale * (A[M,K] W[N,K]^T + bias[N])), A/W bf16 row-major, K and N multiples of 8,
 * act 0 = none / 1 = SiLU, out fp32 (out_f32 = 1) or bf16. */
int egnn_gemm_bf16(int32_t M, int32_t N, int32_t K, const void* A, const void* W, const float* bias,
                   float scale, int32_t act, void* out, int32_t out_f32, void* stream);

/*
 * GlobalLinearAttention of EGNN_Network (reference egnn_pytorch.py:81-144, applied between layers at :445-446): the
 * T global tokens attend over the (masked) nodes, the nodes attend over the induced tokens, residuals, pre-norm GELU
 * feed-forward.  Forward only, fp32 / fp64 (a bf16 module passes fp32 copies).  Weights exactly as the reference's
 * state dict stores them (row-major [out, in]); all pointers device memory, contiguous.
 */
typedef struct EgnnGlobalAttnDesc {
  int32_t abi_version;    /* EGNN_ABI_VERSION */
  int32_t dtype;          /* EGNN_DTYPE_F32 | EGNN_DTYPE_F64 */
  int32_t B, N, T;        /* graphs, nodes, global tokens (T <= 32, else EGNN_ERR_UNSUPPORTED; the Python module
                             GlobalLinearAttention falls back to its PyTorch arithmetic above 32) */
  int32_t dim, heads, dim_head;
} EgnnGlobalAttnDesc;

typedef struct EgnnGlobalAttnWeights {
  const void* norm_seq_g; const void* norm_seq_b;      /* [dim]  norm_seq.weight / .bias        */
  const void* norm_q_g;   const void* norm_q_b;        /* [dim]  norm_queries.weight / .bias    */
  const void* a1_wq;  const void* a1_wkv;              /* [inner, dim], [2 inner, dim]  attn1.to_q / to_kv.weight (inner = heads * dim_head) */
  const void* a1_wo;  const void* a1_bo;               /* [dim, inner], [dim]           attn1.to_out.weight / .bias */
  const void* a2_wq;  const void* a2_wkv; const void* a2_wo; const void* a2_bo;   /* attn2, same shapes */
  const void* ff_ln_g; const void* ff_ln_b;            /* [dim]          ff.0.weight / .bias    */
  const void* ff_w1;  const void* ff_b1;               /* [4 dim, dim], [4 dim]   ff.1          */
  const void* ff_w2;  const void* ff_b2;               /* [dim, 4 dim], [dim]     ff.3          */
} EgnnGlobalAttnWeights;

typedef struct EgnnGlobalAttnIO {
  const void*    x;            /* [B, N, dim] node features                         */
  const void*    queries;      /* [B, T, dim] global tokens                         */
  const uint8_t* mask;         /* [B, N] 0/1 or NULL; a fully masked graph attends uniformly (:101-104) */
  void*          x_out;        /* [B, N, dim]                                       */
  void*          queries_out;  /* [B, T, dim]                                       */
} EgnnGlobalAttnIO;

int egnn_global_attn_workspace_bytes(const EgnnGlobalAttnDesc* desc, size_t* out_bytes);
int egnn_global_attn_forward(const EgnnGlobalAttnDesc* desc, const EgnnGlobalAttnWeights* w, const EgnnGlobalAttnIO* io,
                             void* workspace, size_t workspace_bytes, void* stream);

/*
 * Peer-memory all-gather over NVLink for the ROW-SHARDED single graph (SURVEY.md section 8(e) row 2; reference
 * semantics: the all-pairs pass of egnn_pytorch.py:232-233 runs over ALL nodes, so every rank needs every rank's
 * coordinates and features on the j side).  One process per GPU.  The communicator is the one object of this library
 * that owns device memory beyond a call: a gather buffer (2 x payload_bytes, double-buffered by call parity) that the
 * peers map with CUDA IPC.
 *   egnn_comm_create   -> allocates the buffer on the current device, returns the communicator and a 64-byte IPC handle;
 *                         exchange the handles of all ranks out of band (torch.distributed.all_gather_object) ...
 *   egnn_comm_connect  -> ... and pass all of them (world x 64 bytes, rank order) to map the peers' buffers.
 *   egnn_comm_allgather-> ONE kernel on `stream`: copies this rank's `nseg` segments src[s] (bytes[s], multiples of 4)
 *                         to byte offset dst_off[s] of EVERY rank's buffer with P2P stores over NVLink, raises this rank's
 *                         epoch flag in every peer and waits (on the device) for every peer's flag.  Kernels enqueued
 *                         after it on the same stream see the complete buffer at *gathered_out (valid until the call
 *                         after next).  Every rank must make the same sequence of calls.  No host synchronisation.
 *   egnn_comm_status   -> 0, or 1 if a wait timed out (a peer never arrived); synchronises.
 */
#define EGNN_IPC_HANDLE_BYTES 64
int egnn_comm_create(int32_t world, int32_t rank, size_t payload_bytes, void** comm_out, void* ipc_handle_out);
int egnn_comm_connect(void* comm, const void* all_handles);
int egnn_comm_allgather(void* comm, int32_t nseg, const void* const* src, const size_t* dst_off, const size_t* bytes,
                        void** gathered_out, void* stream);
int egnn_comm_status(void* comm, int32_t* status_out);
int egnn_comm_destroy(void* comm);

/* Diagnostics for benchmarks: when enabled, every egnn_layer_forward brackets its stages
 * (0 neighbour select, 1 per-node tables, 2 fused edge kernel, 3 node update) with CUDA events
 * on the launch stream and counts kernel launches.  egnn_profile_read synchronises those events
 * and returns the accumulated milliseconds / span counts per stage (arrays of 4) and the launch
 * count.  Off by default; the only mutable global state in the library. */
int egnn_profile_enable(int on);
int egnn_profile_read(float* ms_out, int32_t* spans_out, int64_t* launches_out, int reset);

#ifdef __cplusplus
}
#endif
#endif  /* EGNN_B200_H_ */

"""Host-side mirror of the reference's module interface for the EGNN hot path (forward and backward).

`EGNN` and `EGNN_Network` keep the constructor arguments, forward signatures, return values and
state-dict keys of lucidrains/egnn-pytorch (reference egnn_pytorch/egnn_pytorch.py:148-341 and
:343-454), so a reference `state_dict()` loads unchanged -- but `forward` does not execute any
PyTorch arithmetic for the edge step: it packs a POD descriptor and calls the hand-written
sm_90a kernels of libegnn_b200.so through the C ABI (include/egnn_b200.h) on the current CUDA
stream.  PyTorch is used for parameter storage, device memory and streams only.

There is no CPU compute path.  CPU tensors (the reference's own tests pass CPU float64) are
staged to the current CUDA device and the results copied back -- a transport convenience.

Element type -> kernel family
    float64 parameters  -> fp64 SIMT kernels      (parity with the fp64 oracle to ~1e-12)
    float32 parameters  -> fp32 SIMT kernels      ("accurate": the stated-fp32-tolerance path)
    bfloat16 parameters -> bf16 tensor-core kernels (wgmma / mma.sync) with fp32 accumulation ("fast");
                           option combinations the tensor-core kernels do not cover run on the
                           fp32 SIMT kernels instead (still on the GPU; see `last_path`).
`precision='fast'` / `'accurate'` overrides the choice for fp32/bf16 parameters.

Training: when autograd is recording and an input or parameter requires grad, the layer runs as a
`torch.autograd.Function` whose backward is `egnn_layer_backward` -- hand-written recompute-in-backward
kernels (fp32 / fp64; bf16 modules train through the fp32 kernels).  Under `torch.no_grad()` /
`requires_grad_(False)` nothing is saved and the fastest kernels are used.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import os
import types
import warnings
import weakref

import torch
from torch import nn
import torch.nn.functional as F

from . import _native as nat

__all__ = ["EGNN", "EGNN_Network", "CoorsNorm", "GlobalLinearAttention", "edge_index_to_neighbors", "radius_neighbors",
           "radius_neighbors_wide", "knn_neighbors"]


def exists(v):
    return v is not None


# ----------------------------------------------------------------------------- runtime helpers

_WORKSPACES: dict = {}
_NULL_CTX = contextlib.nullcontext()


def _workspace(device: torch.device, nbytes: int, stream_handle=None) -> torch.Tensor:
    """Per-(device, stream) scratch arena, grown on demand; the library never allocates."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream if stream_handle is None else stream_handle)
    ws = _WORKSPACES.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _WORKSPACES[key] = ws
    return ws


class _Built:
    """Stream order of a cache entry: the stream whose work writes the entry's device tensors, and an event recorded on
    it after that work.  A later call on another stream runs `use_on(stream)` first: that stream waits for the event,
    so it never reads the entry before it is written, and the tensors are recorded as in use there (record_stream), so
    the caching allocator does not hand their blocks to the building stream's next allocation while this stream may
    still read them.  Once per entry and stream; a call on the building stream compares two handles and nothing else.
    Nothing synchronises with the host.  An entry built while a CUDA graph is being captured gets no event, and no
    wait is issued during a capture: the graph orders its own replay."""
    __slots__ = ("stream", "event", "tensors", "seen")

    def __init__(self, stream, tensors):
        self.stream, self.tensors, self.seen, self.event = stream.cuda_stream, tensors, set(), None
        if not torch.cuda.is_current_stream_capturing():
            self.event = torch.cuda.Event()
            self.event.record(stream)

    def use_on(self, stream):
        h = stream.cuda_stream
        if self.event is None or h in self.seen or torch.cuda.is_current_stream_capturing():
            return
        stream.wait_event(self.event)
        for t in self.tensors:
            t.record_stream(stream)
        self.seen.add(h)


def _compute_device(t: torch.Tensor) -> torch.device:
    if t.is_cuda:
        return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("egnn_pytorch_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


_KERNEL_DTYPE = {torch.float32: nat.DTYPE_F32, torch.float64: nat.DTYPE_F64, torch.bfloat16: nat.DTYPE_BF16}
_PATH_NAME = {torch.float64: "fp64-simt", torch.float32: "fp32-simt", torch.bfloat16: "bf16-tc"}
# k > 32: knn_block_sort_kernel sorts a row's next_pow2(N) (rank, index) pairs in at most 200 KiB of shared memory
SELECT_SORT_MAX_N = 16384


def _raise_if_sort_limit(err, sort_limited, k, n):
    """A layer with k > 32 that the cell grid does not serve (no mask, no finite valid_radius, N below the grid's
    threshold, ...) ranks each row with a shared-memory sort of all N nodes; the forward rejects such a layer beyond
    SELECT_SORT_MAX_N as unsupported.  That error, and only that one, is reported as the sort's limit."""
    if sort_limited and err.code == nat.ERR_UNSUPPORTED and err.fn.startswith("egnn_layer_forward"):
        raise RuntimeError(f"num_nearest_neighbors={k} > 32 ranks each node with a shared-memory sort of all N nodes, "
                           f"which holds at most N={SELECT_SORT_MAX_N}, got N={n}: use k <= 32, give the layer a mask "
                           f"and a finite valid_radius (the cell grid then selects up to 256 neighbours), or pass "
                           f"neighbors= (e.g. from radius_neighbors_wide); for plain k-nearest lists of any N, build "
                           f"them with knn_neighbors(coors, k, mask=, box=, cell=) and pass neighbors=") from None


def _select_flags(k, n, row_scan):
    """-> (select flags, sort_limited) of a layer that ranks its own k-nearest lists over N nodes (`row_scan`: an
    only_sparse layer with a mask and an adjacency, which ranks nothing).  EGNN_FLAG_CELL_SELECT_WIDE lets a radius
    graph with k > 32 select on the cell grid; otherwise the all-pairs sort ranks each such row, which the library
    rejects beyond SELECT_SORT_MAX_N (sort_limited).  EGNN_FLAG_KNN_GRID lets the library take the same lists from the
    kNN grid where it applies (C <= 3, no adjacency, N at its threshold); a layer beyond the sort's limit keeps its
    error, and knn_neighbors + neighbors= is the way through.  Mask and valid_radius do not enter: the library decides
    from the descriptor and the call."""
    fl, sort_limited = 0, False
    if k > 32:
        fl |= nat.FLAG_CELL_SELECT_WIDE
        sort_limited = n > SELECT_SORT_MAX_N and not row_scan
    if not sort_limited:
        fl |= nat.FLAG_KNN_GRID
    return fl, sort_limited


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _as_u8(t, dev):
    """bool / uint8 / numeric 0-1 tensor -> contiguous, 16-byte aligned uint8 on `dev`, zero-copy when it already is one."""
    if t is None:
        return None
    if t.device != dev:
        t = t.to(dev, non_blocking=True)
    if t.dtype == torch.bool:
        t = t.view(torch.uint8)
    elif t.dtype != torch.uint8:
        t = t.ne(0).view(torch.uint8)
    return t if (t.is_contiguous() and t.data_ptr() % 16 == 0) else t.clone(memory_format=torch.contiguous_format)


def _as(t, dev, dtype):
    """Tensor on `dev` in `dtype`, contiguous and 16-byte aligned (the library's pointer contract, include/egnn_b200.h);
    no work when it already is.  A contiguous view that starts off a 16-byte boundary (a batch slice `x[1:3]`, `x[:, 1:]`
    of a single graph) is copied."""
    if t is None:
        return None
    if t.device == dev and t.dtype == dtype and t.is_contiguous():
        return t.detach() if t.data_ptr() % 16 == 0 else t.detach().clone(memory_format=torch.contiguous_format)
    return t.detach().to(device=dev, dtype=dtype, non_blocking=True).contiguous()


# ----------------------------------------------------------------------------- small modules


class CoorsNorm(nn.Module):
    """Parameter holder for `coors_norm.scale` (reference egnn_pytorch.py:67-77); the
    normalisation x / max(|x|, eps) * scale itself runs inside the fused edge kernel."""

    def __init__(self, eps=1e-8, scale_init=1.0):
        super().__init__()
        self.eps = eps
        self.scale = nn.Parameter(torch.full((1,), float(scale_init)))


def _mlp(d_in, d_hidden, d_out, dropout, final_act=False):
    """Linear -> (Dropout|Identity) -> SiLU -> Linear [-> SiLU]; the Sequential indices (0 and 3)
    are part of the state-dict contract (reference :178-184, :196-201, :203-208)."""
    mods = [nn.Linear(d_in, d_hidden), nn.Dropout(dropout) if dropout > 0 else nn.Identity(), nn.SiLU(),
            nn.Linear(d_hidden, d_out)]
    if final_act:
        mods.append(nn.SiLU())
    return nn.Sequential(*mods)


# ----------------------------------------------------------------------------- autograd bridge


class _EGNNLayerFunction(torch.autograd.Function):
    """forward = egnn_layer_forward on a private workspace that is kept for backward;
    backward = egnn_layer_backward (what autograd derives from reference egnn_pytorch.py:224-341).  `lattice`: the
    caller's box or cell when its gradient was asked for (`lattice_grad=True`), else None; the backward then runs the
    `_lattice` entry point when autograd needs that gradient."""

    @staticmethod
    def forward(ctx, run, feats, coors, edges, label_emb, lattice, *params):
        f_out, x_out, saved = run()
        ctx.saved = saved
        ctx.lattice_dim = None if lattice is None else lattice.dim()
        tensors = (feats, coors, edges, label_emb, lattice) + params
        ctx.meta = [(t.dtype, t.device) if t is not None else None for t in tensors]
        # the saved state aliases the inputs and (same device / dtype) the live parameters: remember their versions so
        # that an in-place edit between forward and backward is reported instead of silently differentiated
        ctx.versions = [(t, t._version) for t in tensors if t is not None]
        return f_out, x_out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_f, g_x):
        sv = ctx.saved
        if sv is None:
            raise RuntimeError("egnn_pytorch_b200: backward through this EGNN layer a second time: the saved forward workspace "
                               "is released after the first backward (retain_graph=True is not supported; run the forward again)")
        for t, v in ctx.versions:
            if t._version != v:
                raise RuntimeError("egnn_pytorch_b200: a tensor needed for the gradient of an EGNN layer (an input or a parameter) "
                                   "was modified in place between forward and backward")
        lib, dev, kdt, cdt = nat.load(), sv["dev"], sv["kdt"], sv["cdt"]
        T = sv["tensors"]
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            g_f, g_x = _as(g_f, dev, kdt), _as(g_x, dev, cdt)
            gw = {f: torch.empty_like(T[f]) for f in nat.WEIGHT_FIELDS if f in T}
            g_feats, g_coors = torch.empty_like(sv["f_in"]), torch.empty_like(sv["x_in"])
            g_edges = torch.empty_like(sv["e_in"]) if (sv["e_in"] is not None and ctx.needs_input_grad[3]) else None
            grads = nat.LayerGrads(g_feats_out=g_f.data_ptr(), g_coors_out=g_x.data_ptr(), g_feats=g_feats.data_ptr(),
                                   g_coors=g_coors.data_ptr(), g_edges=None if g_edges is None else g_edges.data_ptr(),
                                   w=nat.LayerWeightGrads(**{f: t.data_ptr() for f, t in gw.items()}))
            nb = C.c_size_t()
            nat.check("egnn_layer_backward_workspace_bytes",
                      lib.egnn_layer_backward_workspace_bytes(C.byref(sv["desc"]), C.byref(nb)))
            ws = _workspace(dev, nb.value)
            g_lat = None
            if ctx.needs_input_grad[5]:
                # dL/dbox [B, C] or dL/dcell [B, C, C], accumulated by the library in float64
                lat = sv["cell"] if sv["cell"] is not None else sv["box"]
                fn = "egnn_layer_backward_triclinic_lattice" if sv["cell"] is not None else "egnn_layer_backward_periodic_lattice"
                g_lat = torch.empty(lat.shape, dtype=torch.float64, device=dev)
                nat.check(fn, getattr(lib, fn)(C.byref(sv["desc"]), C.byref(sv["w"]), _ptr(sv["packed"]), C.byref(sv["io"]),
                                               _ptr(lat), _ptr(sv["ws"]), C.byref(grads), _ptr(g_lat), _ptr(ws), ws.numel(),
                                               stream))
                if ctx.lattice_dim == lat.dim() - 1:
                    g_lat = g_lat.sum(0)              # one lattice shared by the batch
            elif sv["cell"] is not None:
                nat.check("egnn_layer_backward_triclinic",
                          lib.egnn_layer_backward_triclinic(C.byref(sv["desc"]), C.byref(sv["w"]), _ptr(sv["packed"]),
                                                            C.byref(sv["io"]), _ptr(sv["cell"]), _ptr(sv["ws"]),
                                                            C.byref(grads), _ptr(ws), ws.numel(), stream))
            elif sv["box"] is None:
                nat.check("egnn_layer_backward",
                          lib.egnn_layer_backward(C.byref(sv["desc"]), C.byref(sv["w"]), _ptr(sv["packed"]), C.byref(sv["io"]),
                                                  _ptr(sv["ws"]), C.byref(grads), _ptr(ws), ws.numel(), stream))
            else:
                nat.check("egnn_layer_backward_periodic",
                          lib.egnn_layer_backward_periodic(C.byref(sv["desc"]), C.byref(sv["w"]), _ptr(sv["packed"]),
                                                           C.byref(sv["io"]), _ptr(sv["box"]), _ptr(sv["ws"]), C.byref(grads),
                                                           _ptr(ws), ws.numel(), stream))
            if sv["rows"] is not None:
                # a row block returns its inputs unchanged outside [r0, r1): the identity's gradient for those rows (the
                # library's partial gradients cover the block's own outputs only)
                r0, r1 = sv["rows"]
                for g_in, g_out in ((g_feats, g_f), (g_coors, g_x)):
                    g_in[:, :r0] += g_out[:, :r0]
                    g_in[:, r1:] += g_out[:, r1:]
        ctx.saved = None
        back = lambda g, m: None if (g is None or m is None) else g.to(device=m[1], dtype=m[0])
        out = [None, back(g_feats, ctx.meta[0]), back(g_coors, ctx.meta[1]), back(g_edges, ctx.meta[2]),
               back(gw.get("label_emb"), ctx.meta[3]), back(g_lat, ctx.meta[4])]
        for f, m in zip(sv["param_fields"], ctx.meta[5:]):
            out.append(back(gw.get(f), m))
        return tuple(g if need else None for g, need in zip(out, ctx.needs_input_grad))


# ----------------------------------------------------------------------------- the layer


class EGNN(nn.Module):
    """Drop-in for `egnn_pytorch.EGNN` (reference egnn_pytorch.py:148-341)."""

    def __init__(self, dim, edge_dim=0, m_dim=16, fourier_features=0, num_nearest_neighbors=0, dropout=0.0,
                 init_eps=1e-3, norm_feats=False, norm_coors=False, norm_coors_scale_init=1e-2,
                 update_feats=True, update_coors=True, only_sparse_neighbors=False, valid_radius=float("inf"),
                 m_pool_method="sum", soft_edges=False, coor_weights_clamp_value=None, precision="auto"):
        super().__init__()
        assert m_pool_method in {"sum", "mean"}, "pool method must be either sum or mean"
        assert update_feats or update_coors, "you must update either features, coordinates, or both"
        assert precision in {"auto", "accurate", "fast"}
        self.dim, self.edge_dim, self.m_dim = dim, edge_dim, m_dim
        self.fourier_features = fourier_features
        edge_input_dim = fourier_features * 2 + dim * 2 + edge_dim + 1
        self.edge_mlp = _mlp(edge_input_dim, edge_input_dim * 2, m_dim, dropout, final_act=True)
        self.edge_gate = nn.Sequential(nn.Linear(m_dim, 1), nn.Sigmoid()) if soft_edges else None
        self.node_norm = nn.LayerNorm(dim) if norm_feats else nn.Identity()
        self.coors_norm = CoorsNorm(scale_init=norm_coors_scale_init) if norm_coors else nn.Identity()
        self.m_pool_method = m_pool_method
        self.node_mlp = _mlp(dim + m_dim, dim * 2, dim, dropout) if update_feats else None
        self.coors_mlp = _mlp(m_dim, m_dim * 4, 1, dropout) if update_coors else None
        self.num_nearest_neighbors = num_nearest_neighbors
        self.only_sparse_neighbors = only_sparse_neighbors
        self.valid_radius = valid_radius
        self.coor_weights_clamp_value = coor_weights_clamp_value
        self.dropout_p = dropout
        self.init_eps = init_eps
        self.precision = precision
        self.last_path = None          # 'fp64-simt' | 'fp32-simt' | 'bf16-tc' of the last call
        self.cache_policy = "version"  # 'version' | 'always' -- see invalidate_cache()
        self._stage = {}
        self._tc_unsupported = set()
        self._call_cache = {}
        self.apply(self._init)

    def _init(self, module):
        if type(module) is nn.Linear:
            nn.init.normal_(module.weight, std=self.init_eps)      # reference :219-222

    # -------------------------------------------------------------- parameter staging
    def _state_fields(self):
        """[(EgnnLayerWeights field, Parameter)], cached; rebuilt if a Parameter object is replaced."""
        cache = self.__dict__.get("_fields_cache")
        if cache is not None and all(mod._parameters.get(name) is p for mod, name, _, p in cache):
            return cache
        cache = []
        for mname, mod in self.named_modules():
            for pname, p in mod._parameters.items():
                key = f"{mname}.{pname}" if mname else pname
                f = nat.STATE_KEY_TO_FIELD.get(key)
                if f is not None and p is not None:
                    cache.append((mod, pname, f, p))
        self.__dict__["_fields_cache"] = cache
        return cache

    def invalidate_cache(self):
        """Drop every staged / packed copy of the parameters (they are rebuilt on the next call).

        The caches are keyed on (storage pointer, tensor version) of each parameter.  Writes that go THROUGH
        `.data` (`p.data.copy_(master)`, the master->model copy of apex / DeepSpeed / Megatron-style mixed
        precision, some EMA loops) do not bump the version counter, so after such a write call this method -- or
        set `cache_policy = "always"` to re-stage and re-pack on every forward (one small kernel per layer).
        In training mode (`module.training` with a parameter that requires grad) the layer always re-packs."""
        self._stage = {}
        self._call_cache = {}
        self.__dict__.pop("_fields_cache", None)

    def _staged(self, device, dtype):
        """-> the staged entry for (device, dtype).  A new entry's "built" (its stream order, `_Built`) is set by _run
        once its packed parameters are enqueued: one call, on one stream, writes its copies, label table and pack."""
        fields = self._state_fields()
        sig = [x for _, _, _, p in fields for x in (p.data_ptr(), p._version)]
        key = (device, dtype)
        st = self._stage.get(key)
        always = self.cache_policy == "always" or (self.training and any(p.requires_grad for _, _, _, p in fields))
        if st is None or st["sig"] != sig or always:
            with torch.no_grad():
                tensors = {f: p.detach().to(device=device, dtype=dtype).contiguous() for _, _, f, p in fields}
            st = dict(sig=sig, tensors=tensors, packed={}, wstruct={}, built=None)
            self._stage[key] = st
        return st

    def _flags(self):
        fl = self.__dict__.get("_flags_cache")
        if fl is None:                           # which sub-modules exist is fixed by the constructor
            fl = 0
            if isinstance(self.node_norm, nn.LayerNorm): fl |= nat.FLAG_NORM_FEATS
            if isinstance(self.coors_norm, CoorsNorm): fl |= nat.FLAG_NORM_COORS
            if self.node_mlp is not None: fl |= nat.FLAG_UPDATE_FEATS
            if self.coors_mlp is not None: fl |= nat.FLAG_UPDATE_COORS
            if self.edge_gate is not None: fl |= nat.FLAG_SOFT_EDGES
            self.__dict__["_flags_cache"] = fl
        # plain attributes a user may change between calls are read every time
        if self.m_pool_method == "mean": fl |= nat.FLAG_POOL_MEAN
        if self.coor_weights_clamp_value is not None: fl |= nat.FLAG_CLAMP
        return fl

    def _kernel_dtype(self):
        pd = self._modules["edge_mlp"]._modules["0"]._parameters["weight"].dtype     # edge_mlp[0].weight without three __getattr__ hops
        if pd == torch.float64:
            return torch.float64
        prec = os.environ.get("EGNN_B200_PRECISION", self.precision)
        if prec == "fast" or (prec == "auto" and pd == torch.bfloat16):
            return torch.bfloat16
        return torch.float32

    # -------------------------------------------------------------- forward
    def forward(self, feats, coors, edges=None, mask=None, adj_mat=None, *, neighbors=None, neighbor_edges=None, box=None,
                cell=None, lattice_grad=False, ptr=None, _edge_labels=None, _label_emb=None, _k_hint=None, _rows=None):
        """Reference signature `forward(feats, coors, edges=None, mask=None, adj_mat=None)` (egnn_pytorch.py:224).

        `neighbors` (additive, keyword-only): int tensor [B, N, k] of neighbour indices, -1 = empty slot.  When
        given, the layer runs on exactly these edges and the O(N^2) distance / top-k pass is skipped -- the
        edge-list mode of SURVEY.md section 8(f) (`edge_index_to_neighbors` converts a PyG-style edge_index).

        `neighbor_edges` (additive, keyword-only, needs `neighbors`, replaces `edges`): float tensor
        [B, N, k, edge_dim] of edge features per neighbour slot -- slot s of node i holds the features of the edge
        neighbors[b, i, s] -> i -- so a sparse graph needs no [B, N, N, edge_dim] tensor.  Its gradient has the same
        shape (0 in empty slots).

        `box` (additive, keyword-only): periodic boundaries.  Float tensor of box lengths, [C] (shared by the batch) or
        [B, C], on any device; every pair geometry x_i - x_j becomes its minimum image rel - L rint(rel / L) on the axes
        with a finite L > 0 (L = 0 or inf: not periodic).  Distances, neighbour ranking, CoorsNorm and the coordinate
        update follow; the output coordinates are not wrapped back into the box.  Orthorhombic boxes, one image per
        neighbour.  A box that requires grad is rejected unless `lattice_grad=True`.

        `cell` (additive, keyword-only, instead of `box`): periodic boundaries in a triclinic cell.  Float tensor [C, C]
        (shared by the batch) or [B, C, C], C in {2, 3}, row k = lattice vector a_k, lower-triangular (the LAMMPS
        restricted-triclinic form; README shows how to rotate any cell into it).  A diagonal entry of 0 or inf leaves
        its axis aperiodic; that axis's row and column must be zero off the diagonal.  Every pair vector is wrapped
        sequentially from the last axis to the first (n = rint(r_c / L_c), r_d -= cell[c, d] n for d <= c), after which
        |r_c| <= L_c / 2 on every periodic axis: the result lies in the centred box of the diagonal entries, a
        fundamental domain of the lattice, so it is the minimum image whenever the minimum image is shorter than
        min_c L_c / 2; pairs farther apart get that centred-box image, one image per neighbour.  A diagonal cell gives
        exactly the outputs of `box=` with the same lengths.  A cell that requires grad is rejected unless
        `lattice_grad=True`.

        `lattice_grad` (additive, keyword-only, needs `box` or `cell`): accept a box / cell that requires grad and give
        it its gradient through autograd, for stress and virial (README).  The wrap is rel = (x_i - x_j) - sum_c n_c a_c
        with integer image counts n, so dL/dcell[c, d] = -sum_pairs n_c dL/drel_d for d <= c (0 above the diagonal),
        dL/dbox[c] = -sum_pairs n_c dL/drel_c, and 0 on aperiodic axes; neighbour selection contributes nothing.  A [C] /
        [C, C] lattice gets the sum over the batch.  No effect under torch.no_grad().

        `ptr` (additive, keyword-only): a packed batch of variable-size graphs, PyTorch Geometric's layout.  feats
        [1, T, dim] and coors [1, T, C] hold G graphs end to end, graph g on nodes ptr[g] .. ptr[g+1]-1 of the 1-D integer
        tensor ptr [G+1] (ptr[0] = 0, non-decreasing, ptr[G] = T; any device).  Every graph gets what it would get
        alone, to the rounding of the kernel type: with num_nearest_neighbors = k, its k nearest nodes of its own
        graph (all of its nodes, with mean pooling over them, when it has fewer than k); without, all of its nodes
        (dense).  The lists are ranked on the device as each graph's unpacked call would rank them: on the radius grid
        (a mask and 0 < valid_radius < 1e5) or the kNN grid for graphs of at least EGNN_B200_CELL_SELECT_MIN_N /
        EGNN_B200_KNN_GRID_MIN_N nodes (C <= 3), in O(n_g); otherwise by the segmented all-pairs select in O(n_g^2) --
        the cost of each graph alone, not of the batch padded to its largest graph.  The lists are the same either
        way, and the layer runs on them in edge-list mode, forward and backward.  `mask` [1, T] and one `box` [C] or `cell` [C, C] shared by every graph
        combine with it; per-graph lattices, `neighbors`, `neighbor_edges`, dense `edges`, adjacency and
        only_sparse_neighbors do not (ValueError).  ptr's values are read on the host once per tensor version."""
        if ptr is not None:
            neighbors, mask = self._packed_lists(feats, coors, ptr, edges, mask, adj_mat, neighbors, neighbor_edges, box,
                                                 cell, _edge_labels, _rows)
        if neighbor_edges is not None:
            edges = self._check_neighbor_edges(feats, edges, neighbors, neighbor_edges, _label_emb)
        lattice = _check_lattice(box, cell, feats.shape[0], coors.shape[-1], self.__dict__, lattice_grad)
        if torch.is_grad_enabled():             # (the parameter scan is skipped entirely under torch.no_grad())
            fields = self._state_fields()
            if (feats.requires_grad or coors.requires_grad or (edges is not None and edges.requires_grad) or
                    (_label_emb is not None and _label_emb.requires_grad) or any(p.requires_grad for _, _, _, p in fields) or
                    (lattice is not None and lattice.requires_grad)):
                return self._forward_train(fields, feats, coors, edges, mask, adj_mat, neighbors, _edge_labels, _label_emb,
                                           _k_hint, _rows, neighbor_edges is not None, box, cell, lattice)
            with torch.no_grad():
                return self._forward_impl(feats, coors, edges, mask, adj_mat, neighbors, _edge_labels, _label_emb, _k_hint,
                                          _rows, slot_edges=neighbor_edges is not None, box=box, cell=cell)
        return self._forward_impl(feats, coors, edges, mask, adj_mat, neighbors, _edge_labels, _label_emb, _k_hint, _rows,
                                  slot_edges=neighbor_edges is not None, box=box, cell=cell)

    def _packed_lists(self, feats, coors, ptr, edges, mask, adj_mat, neighbors, neighbor_edges, box, cell, labels, rows):
        """forward(ptr=): the checks (ValueError before anything launches), then -> (neighbour lists [1, T, k], the mask
        edge-list mode runs with).  kNN: the segmented select's lists; under a caller's mask its ok = 0 slots (rank above
        valid_radius) are emptied, as the per-graph select's ok bytes drop them there (without a mask the layer keeps
        every slot, and so do these lists).  Dense: every node of the node's own graph.  Slots past a graph's size are
        -1.  List mode runs with the caller's mask or with an all-ones one, so that mean pooling divides by the slots
        the graph fills, as the per-graph call does."""
        for bad, what in ((neighbors is not None or neighbor_edges is not None, "neighbors= / neighbor_edges= (the lists "
                           "already define the graphs)"),
                          (edges is not None, "dense edges [B, N, N, edge_dim]"),
                          (adj_mat is not None or labels is not None or self.only_sparse_neighbors,
                           "adj_mat, only_sparse_neighbors or num_adj_degrees"),
                          (rows is not None, "a row range (_rows)")):
            if bad:
                raise ValueError(f"ptr= (a packed batch) cannot be combined with {what}")
        t, c = coors.shape[1], coors.shape[-1]
        if feats.shape[:2] != coors.shape[:2]:
            raise ValueError(f"feats and coors must hold the same [1, T] nodes, got {tuple(feats.shape)} and "
                             f"{tuple(coors.shape)}")
        max_n = _check_ptr(ptr, coors.shape[0], t)
        _check_packed_lattice(box, cell)
        dev = _compute_device(feats)
        with _NULL_CTX if torch.cuda.current_device() == dev.index else torch.cuda.device(dev):
            m = _as_u8(mask, dev)
            if self.num_nearest_neighbors > 0:
                cdt = torch.float64 if self._kernel_dtype() == torch.float64 else torch.float32   # as the layer's select
                # a masked layer with a radius the radius grid serves keeps only in-radius slots: radius mode
                mode = "radius" if m is not None and _in_cell_radius(self.valid_radius, cdt) else "knn"
                idx, ok = _packed_select(_as(coors, dev, cdt), ptr, min(self.num_nearest_neighbors, max_n), m,
                                         _packed_lattice(box, cell, dev, cdt, c), cell is not None, self.valid_radius,
                                         mode, max_n)
                lists = idx if m is None else idx.masked_fill(ok == 0, -1)
            else:
                lists = _dense_packed_lists(ptr, t, max_n, dev)
            run_mask = mask if mask is not None else torch.ones((1, t), dtype=torch.bool, device=dev)
        return lists, run_mask

    def _check_neighbor_edges(self, feats, edges, neighbors, neighbor_edges, label_emb):
        """Misuse of `neighbor_edges` raises here, before anything is staged or launched; -> the tensor to run with."""
        if neighbors is None:
            raise ValueError("neighbor_edges needs neighbors=: its slots follow the caller's neighbour lists")
        if edges is not None:
            raise ValueError("pass edge features either as edges [B, N, N, edge_dim] or as neighbor_edges "
                             "[B, N, k, edge_dim], not both")
        edge_dim = self.edge_dim - (0 if label_emb is None else label_emb.shape[1])
        b, n = feats.shape[:2]
        want = (b, n, neighbors.shape[-1], edge_dim)
        if edge_dim == 0 or tuple(neighbor_edges.shape) != want or not neighbor_edges.is_floating_point():
            raise ValueError(f"neighbor_edges must be a float tensor of shape (B, N, k, edge_dim) = {want} for this layer "
                             f"(edge_dim > 0), got {neighbor_edges.dtype} {tuple(neighbor_edges.shape)}")
        return neighbor_edges

    def _forward_train(self, fields, feats, coors, edges, mask, adj_mat, neighbors, labels, label_emb, k_hint, rows,
                       slot_edges=False, box=None, cell=None, lattice=None):
        """With a row range (`_rows=(r0, r1)`) the layer is differentiated as the function it returns: rows r0:r1 are the
        layer's output, every other row is its input unchanged.  The library's backward then yields this block's share
        of every gradient (EGNN_FLAG_ROW_PARTIAL_GRADS): the blocks of a partition of the rows sum to the full gradient."""
        params = [p for _, _, _, p in fields]

        def run():
            return self._forward_impl(feats, coors, edges, mask, adj_mat, neighbors, labels, label_emb, k_hint, rows,
                                      train=True, param_fields=[f for _, _, f, _ in fields], slot_edges=slot_edges, box=box,
                                      cell=cell)

        return _EGNNLayerFunction.apply(run, feats, coors, edges, label_emb, lattice, *params)

    def _forward_impl(self, feats, coors, edges, mask, adj_mat, neighbors, _edge_labels, _label_emb, _k_hint, _rows,
                      train=False, param_fields=None, slot_edges=False, box=None, cell=None):
        """`slot_edges`: `edges` holds features per neighbour slot, [B, N, k, edge_dim] (forward's `neighbor_edges`)."""
        lib = nat.load()
        dev = _compute_device(feats)
        b, n, d = feats.shape
        assert d == self.dim, f"feature width {d} != dim {self.dim}"
        c = coors.shape[-1]
        kdt = self._kernel_dtype()
        # nn.Dropout of the three MLPs (reference :176-208) is active in training mode only, grad or no grad -- like
        # the reference.  The kernels regenerate the masks from (seed, element index) in forward and backward; the seed
        # is drawn per call from torch's CPU generator, so torch.manual_seed makes a run reproducible.
        drop_p = float(self.dropout_p) if (self.training and self.dropout_p > 0) else 0.0
        if (train or drop_p > 0) and kdt == torch.bfloat16:
            kdt = torch.float32                 # the tensor-core kernels are forward-only and have no dropout
        label_dim = 0 if _label_emb is None else _label_emb.shape[1]
        cont_edge_dim = self.edge_dim - label_dim
        assert (edges is None) == (cont_edge_dim == 0), "edges must be given iff edge_dim > 0"

        use_nearest = self.num_nearest_neighbors > 0 or self.only_sparse_neighbors          # reference :230
        adj_u8 = None
        sort_limited = False
        k = 0
        flags = self._flags()
        if slot_edges:
            flags |= nat.FLAG_EDGES_PER_SLOT
        if train and _rows is not None:
            flags |= nat.FLAG_ROW_PARTIAL_GRADS          # backward of the row block only; per-pair buffers sized by it
        nbr = None
        if neighbors is not None:
            assert neighbors.dim() == 3 and neighbors.shape[:2] == (b, n), "neighbors must be [B, N, k]"
            nbr = neighbors.to(device=dev, dtype=torch.int32).contiguous()
            k = nbr.shape[-1]
            if not (0 < k <= n):
                raise RuntimeError(f"neighbour lists need 0 < k <= N, got k={k}, N={n}")
        elif use_nearest:
            k = self.num_nearest_neighbors
            if exists(adj_mat):
                adj_u8 = _as_u8(adj_mat, dev)
                if adj_u8.dim() == 3:
                    flags |= nat.FLAG_ADJ_BATCHED
                if self.only_sparse_neighbors:
                    flags |= nat.FLAG_ONLY_SPARSE                                    # valid_radius := 0 (:250)
                    # reference :249 -- one host sync, diagonal still counted
                    k = int(_k_hint) if _k_hint is not None else int(adj_u8.sum(dim=-1, dtype=torch.int32).max().item())
            if not (0 < k <= n):
                raise RuntimeError(f"number of neighbours k={k} must satisfy 0 < k <= N={n} (torch.topk would raise)")
            row_scan = self.only_sparse_neighbors and exists(mask) and adj_u8 is not None     # no ranking (select_neighbors)
            sel_flags, sort_limited = _select_flags(k, n, row_scan)
            flags |= sel_flags

        # support does not depend on the list length (any k > 0 runs the tensor cores), so one cached "unsupported"
        # entry for all k > 32 stays correct
        cfg_key = (c, k > 0, min(k, 33), cont_edge_dim, label_dim, _rows is None)
        if kdt == torch.bfloat16 and cfg_key in self._tc_unsupported:
            kdt = torch.float32
        try:
            return self._run(lib, dev, kdt, feats, coors, edges, mask, adj_u8, _edge_labels, _label_emb,
                             b, n, c, k, flags, cont_edge_dim, label_dim, _rows, nbr, train, param_fields, drop_p, box, cell)
        except nat.EgnnNativeError as e:
            _raise_if_sort_limit(e, sort_limited, k, n)
            if e.code != nat.ERR_UNSUPPORTED or kdt != torch.bfloat16:
                raise
        # the tensor-core kernels do not cover this option set: fp32 SIMT kernels (still on the GPU); remembered
        self._tc_unsupported.add(cfg_key)
        warnings.warn(f"egnn_pytorch_b200: the bf16 tensor-core kernels do not cover this configuration (C={c}, k={k}, "
                      f"edge_dim={cont_edge_dim}, label_dim={label_dim}, m_dim={self.m_dim}, fourier={self.fourier_features}); "
                      f"running the fp32 SIMT kernels instead (about 5x slower, same results to fp32 accuracy)", UserWarning,
                      stacklevel=3)
        try:
            return self._run(lib, dev, torch.float32, feats, coors, edges, mask, adj_u8, _edge_labels, _label_emb,
                             b, n, c, k, flags, cont_edge_dim, label_dim, _rows, nbr, box=box, cell=cell)
        except nat.EgnnNativeError as e:
            _raise_if_sort_limit(e, sort_limited, k, n)
            raise

    def _run(self, lib, dev, kdt, feats, coors, edges, mask, adj_u8, labels, label_emb, b, n, c, k, flags,
             cont_edge_dim, label_dim, rows, nbr=None, train=False, param_fields=None, drop_p=0.0, box=None, cell=None):
        cdt = torch.float64 if kdt == torch.float64 else torch.float32
        cs = torch.cuda.current_stream(dev)
        stream_handle = cs.cuda_stream
        st = self._staged(dev, kdt)
        built = st["built"]
        if built is not None and built.stream != stream_handle:
            built.use_on(cs)                     # an entry another stream built (None: this call builds it)
        T = dict(st["tensors"])
        lab_w = None
        if label_emb is not None:
            lab_w = st.get("lab_keepalive")
            if lab_w is None or st.get("lab_sig") != (label_emb.data_ptr(), label_emb._version):
                lab_w = label_emb.detach().to(device=dev, dtype=kdt).contiguous()
                st["lab_sig"] = (label_emb.data_ptr(), label_emb._version)
                st["wstruct"] = {}
                st["packed"] = {}
            T["label_emb"] = lab_w

        ckey = (kdt, b, n, c, k, flags, cont_edge_dim, label_dim, 0 if label_emb is None else label_emb.shape[0], rows,
                float(self.valid_radius), float(self.coor_weights_clamp_value or 0.0))
        cc = self._call_cache.get(ckey)
        if cc is None:
            r_lo, r_hi = (0, 0) if rows is None else rows
            if rows is not None and r_lo == r_hi:
                r_lo = r_hi = n                          # an empty block (the descriptor's 0, 0 means all rows)
            desc = nat.LayerDesc(
                abi_version=nat.ABI_VERSION, dtype=_KERNEL_DTYPE[kdt], B=b, N=n, C=c, dim=self.dim,
                edge_dim=cont_edge_dim, label_dim=label_dim, num_labels=0 if label_emb is None else label_emb.shape[0],
                m_dim=self.m_dim, fourier=self.fourier_features, k=k, flags=flags,
                valid_radius=float(self.valid_radius), clamp=float(self.coor_weights_clamp_value or 0.0),
                row_begin=r_lo, row_end=r_hi, reserved=0,
                dropout_p=0.0, dropout_seed=0)
            nb = C.c_size_t()
            nat.check("egnn_layer_workspace_bytes", lib.egnn_layer_workspace_bytes(C.byref(desc), C.byref(nb)))
            cc = (desc, nb.value)
            if len(self._call_cache) > 64:
                self._call_cache.clear()
            self._call_cache[ckey] = cc
        desc, ws_bytes = cc
        if drop_p > 0:                               # per-call copy: fresh seed, kept with the saved state for backward
            d2 = nat.LayerDesc()
            C.memmove(C.byref(d2), C.byref(desc), C.sizeof(nat.LayerDesc))
            d2.dropout_p = drop_p
            d2.dropout_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            desc = d2
        wkey = None if lab_w is None else (label_emb.data_ptr(), label_emb._version)
        w = st["wstruct"].get(wkey)
        if w is None:
            w = nat.LayerWeights(**{f: (T[f].data_ptr() if f in T else None) for f in nat.WEIGHT_FIELDS})
            st["wstruct"] = {wkey: w}
            st["lab_keepalive"] = lab_w

        stream = C.c_void_p(stream_handle)
        ctx = _NULL_CTX if torch.cuda.current_device() == dev.index else torch.cuda.device(dev)
        with ctx:
            # packed parameters, cached until a parameter changes
            pkey = (label_dim, 0 if lab_w is None else (label_emb.data_ptr(), label_emb._version))
            packed = st["packed"].get(pkey)
            if packed is None:
                nb = C.c_size_t()
                nat.check("egnn_layer_packed_bytes", lib.egnn_layer_packed_bytes(C.byref(desc), C.byref(nb)))
                packed = torch.empty(nb.value, dtype=torch.uint8, device=dev)
                nat.check("egnn_layer_pack_weights",
                          lib.egnn_layer_pack_weights(C.byref(desc), C.byref(w), _ptr(packed), nb.value, stream))
                st["packed"] = {pkey: packed}
                st["built"] = _Built(cs, list(T.values()) + [packed])       # the staged copies, label table and pack

            f_in, x_in, e_in = _as(feats, dev, kdt), _as(coors, dev, cdt), _as(edges, dev, kdt)
            bx = None if box is None else _as(box, dev, cdt).expand(b, c).contiguous()     # [B, C], like coors
            if train and bx is not None and bx.data_ptr() == box.data_ptr():
                bx = bx.clone()                  # the backward must see the forward's box, whatever the caller does to it
            cl = None if cell is None else _as(cell, dev, cdt).expand(b, c, c).contiguous()    # [B, C, C]
            if train and cl is not None and cl.data_ptr() == cell.data_ptr():
                cl = cl.clone()                  # (the same for the cell)
            m_in, l_in = _as_u8(mask, dev), _as_u8(labels, dev)
            f_out = torch.empty_like(f_in)
            x_out = torch.empty_like(x_in)
            if rows is not None:       # rows outside the range keep the input values
                f_out.copy_(f_in)
                x_out.copy_(x_in)
            # training: keep the per-pair pre-activations of edge_mlp's second SiLU (64 B per pair in fp32) so
            # that backward need not recompute them, unless that exceeds EGNN_B200_SAVE_PAIR_MB (default 1024).  A row
            # block keeps the pairs of its own rows only: [B, r1 - r0, J, MP]
            pre2 = None
            if train:
                mp = 16 if self.m_dim <= 16 else 32
                n_rows = n if rows is None else rows[1] - rows[0]
                nbytes = b * n_rows * (k if k > 0 else n) * mp * f_in.element_size()
                if nbytes <= float(os.environ.get("EGNN_B200_SAVE_PAIR_MB", "1024")) * 2 ** 20:
                    pre2 = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            # the library reads EgnnLayerIO during the call only: inference re-fills one struct per layer, training
            # (which keeps it with the saved state) gets its own
            io = nat.LayerIO() if train else self.__dict__.get("_io_scratch")
            if io is None:
                io = self.__dict__["_io_scratch"] = nat.LayerIO()
            io.feats = f_in.data_ptr(); io.coors = x_in.data_ptr()
            io.edges = None if e_in is None else e_in.data_ptr()
            io.edge_labels = None if l_in is None else l_in.data_ptr()
            io.mask = None if m_in is None else m_in.data_ptr()
            io.adj = None if adj_u8 is None else adj_u8.data_ptr()
            io.feats_out = f_out.data_ptr(); io.coors_out = x_out.data_ptr()
            io.nbr_idx = None if nbr is None else nbr.data_ptr()
            io.pre2_out = None if pre2 is None else pre2.data_ptr()
            if train:     # preflight: configurations the backward kernels cannot run fail HERE, before the forward launches
                nbb = C.c_size_t()
                nat.check("egnn_layer_backward_workspace_bytes", lib.egnn_layer_backward_workspace_bytes(C.byref(desc), C.byref(nbb)))
            # training keeps the workspace (per-node tables, pooled messages, neighbour lists) for backward
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if train else _workspace(dev, ws_bytes, stream_handle)
            if train or rows is None or rows[0] != rows[1]:      # an empty row block computes nothing in inference
                if cl is not None:
                    nat.check("egnn_layer_forward_triclinic",
                              lib.egnn_layer_forward_triclinic(C.byref(desc), C.byref(w), _ptr(packed), C.byref(io),
                                                               _ptr(cl), _ptr(ws), ws.numel(), stream))
                elif bx is None:
                    nat.check("egnn_layer_forward",
                              lib.egnn_layer_forward(C.byref(desc), C.byref(w), _ptr(packed), C.byref(io), _ptr(ws),
                                                     ws.numel(), stream))
                else:
                    nat.check("egnn_layer_forward_periodic",
                              lib.egnn_layer_forward_periodic(C.byref(desc), C.byref(w), _ptr(packed), C.byref(io), _ptr(bx),
                                                              _ptr(ws), ws.numel(), stream))
        object.__setattr__(self, "last_path", _PATH_NAME[kdt])
        outs = (f_out if (f_out.dtype == feats.dtype and f_out.device == feats.device) else f_out.to(device=feats.device, dtype=feats.dtype),
                x_out if (x_out.dtype == coors.dtype and x_out.device == coors.device) else x_out.to(device=coors.device, dtype=coors.dtype))
        if not train:
            return outs
        saved = dict(dev=dev, kdt=kdt, cdt=cdt, desc=desc, w=w, packed=packed, io=io, ws=ws, tensors=T,
                     f_in=f_in, x_in=x_in, e_in=e_in, param_fields=param_fields, rows=rows, box=bx, cell=cl,
                     keep=(m_in, l_in, adj_u8, nbr, lab_w, pre2))      # everything io points at stays alive
        return outs + (saved,)


def _check_lattice(box, cell, b, c, cache, lattice_grad):
    """The checks of `box=` / `cell=` and `lattice_grad=` -> the box or cell whose gradient is asked for, else None."""
    if box is not None:
        if cell is not None:
            raise ValueError("pass either box= or cell=, not both")
        _check_box(box, b, c, cache, lattice_grad)
    if cell is not None:
        _check_cell(cell, b, c, cache, lattice_grad)
    if not lattice_grad:
        return None
    if box is None and cell is None:
        raise ValueError("lattice_grad=True needs box= or cell=: it asks for the gradient with respect to the lattice")
    return box if box is not None else cell


def _check_box(box, b, c, cache, lattice_grad=False):
    """Misuse of `box=` raises ValueError here, before anything launches.  The value check (no negative or NaN length)
    reads the box on the host.  It is skipped for the very tensor object this module checked last, unchanged since (the
    same object alive and the same version counter: an in-place write bumps it, a write through `.data` does not), and
    while a CUDA graph is being captured (GraphedForward checks the box in its warm-up calls)."""
    if not torch.is_tensor(box) or not box.is_floating_point():
        raise ValueError(f"box must be a float tensor of box lengths, got {type(box).__name__}"
                         f"{'' if not torch.is_tensor(box) else ' ' + str(box.dtype)}")
    if tuple(box.shape) not in ((c,), (b, c)):
        raise ValueError(f"box must have shape (C,) = ({c},) or (B, C) = ({b}, {c}), got {tuple(box.shape)}")
    if box.requires_grad and not lattice_grad:
        raise ValueError("box.requires_grad is set: pass lattice_grad=True for the gradient with respect to the box "
                         "(stress / virial), or box.detach()")
    last = cache.get("_box_checked")
    if last is not None and last[0]() is box and last[1] == box._version:
        return
    if box.is_cuda and torch.cuda.is_current_stream_capturing():
        return
    if bool(((box < 0) | torch.isnan(box)).any()):
        raise ValueError("box lengths must be >= 0 or +inf (0 or inf: the axis is not periodic), got negative or NaN values")
    cache["_box_checked"] = (weakref.ref(box), box._version)


def _check_cell(cell, b, c, cache, lattice_grad=False):
    """Misuse of `cell=` raises ValueError here, before anything launches, with the caching and capture rules of
    _check_box: the value checks read the cell on the host, except for the very tensor object this module checked last,
    unchanged since, and while a CUDA graph is being captured."""
    if not torch.is_tensor(cell) or not cell.is_floating_point():
        raise ValueError(f"cell must be a float tensor of lattice vectors, got {type(cell).__name__}"
                         f"{'' if not torch.is_tensor(cell) else ' ' + str(cell.dtype)}")
    if c not in (2, 3):
        raise ValueError(f"cell= needs C = 2 or 3 coordinates, got C={c}")
    if tuple(cell.shape) not in ((c, c), (b, c, c)):
        raise ValueError(f"cell must have shape (C, C) = ({c}, {c}) or (B, C, C) = ({b}, {c}, {c}), got {tuple(cell.shape)}")
    if cell.requires_grad and not lattice_grad:
        raise ValueError("cell.requires_grad is set: pass lattice_grad=True for the gradient with respect to the cell "
                         "(stress / virial), or cell.detach()")
    last = cache.get("_cell_checked")
    if last is not None and last[0]() is cell and last[1] == cell._version:
        return
    if cell.is_cuda and torch.cuda.is_current_stream_capturing():
        return
    m = cell.detach().to("cpu", torch.float64).reshape(-1, c, c)
    diag = torch.diagonal(m, dim1=-2, dim2=-1)
    off = m.masked_fill(torch.eye(c, dtype=torch.bool), 0.0)
    if bool((torch.triu(m, diagonal=1) != 0).any()):
        raise ValueError("cell must be lower-triangular (row k = lattice vector a_k, cell[k, d] == 0 for d > k); "
                         "rotate a general cell into that form (README, periodic boundaries)")
    if not bool(torch.isfinite(off).all()):
        raise ValueError("cell off-diagonal entries must be finite, got NaN or inf")
    if bool(((diag < 0) | torch.isnan(diag)).any()):
        raise ValueError("cell diagonal entries must be >= 0 or +inf (0 or inf: the axis is not periodic), "
                         "got negative or NaN values")
    aper = (diag == 0) | torch.isinf(diag)                       # [G, C]
    if bool(((off != 0) & (aper.unsqueeze(-1) | aper.unsqueeze(-2))).any()):
        raise ValueError("an aperiodic axis of the cell (diagonal 0 or inf) must have a zero row and column off the "
                         "diagonal")
    cache["_cell_checked"] = (weakref.ref(cell), cell._version)


_PTR_CHECKED: dict = {}


def _check_ptr(ptr, b, t):
    """The checks of `ptr=` (ValueError before anything launches) -> max n_g, the node count of the largest graph.
    ptr is a 1-D integer tensor of G + 1 >= 2 graph offsets on any device, with ptr[0] == 0, non-decreasing and
    ptr[-1] == T, for inputs of B == 1 row of T nodes.  The value checks read ptr on the host once per tensor object
    and version (the caching rule of _check_box, shared by every module and builder), so a repeated call, or a CUDA
    graph that replays one, does not synchronise; a ptr that was never checked cannot be checked inside a capture."""
    if (not torch.is_tensor(ptr) or ptr.dim() != 1 or ptr.numel() < 2 or ptr.is_floating_point() or ptr.is_complex()
            or ptr.dtype == torch.bool):
        raise ValueError(f"ptr must be a 1-D integer tensor of G + 1 >= 2 graph offsets, got "
                         f"{type(ptr).__name__ if not torch.is_tensor(ptr) else f'{ptr.dtype} {tuple(ptr.shape)}'}")
    if b != 1:
        raise ValueError(f"ptr= takes a packed batch: inputs of shape [1, T, ...] with the graphs end to end, got B={b}")
    hit = _PTR_CHECKED.get(id(ptr))
    if hit is not None and hit[0]() is ptr and hit[1] == ptr._version and hit[2] == t:
        return hit[3]
    if ptr.is_cuda and torch.cuda.is_current_stream_capturing():
        raise ValueError("ptr= is checked on the host, which a CUDA graph capture cannot do: run the call once before "
                         "capturing it (GraphedForward's warm-up does)")
    p = ptr.detach().to("cpu", torch.int64)
    if int(p[0]) != 0 or int(p[-1]) != t or bool((p[1:] < p[:-1]).any()):
        raise ValueError(f"ptr must start at 0, be non-decreasing and end at T = {t} (the node count), got "
                         f"{p.tolist() if p.numel() <= 16 else f'{p[:8].tolist()} ... {p[-8:].tolist()}'}")
    max_n = int((p[1:] - p[:-1]).max())
    if len(_PTR_CHECKED) >= 64:
        _PTR_CHECKED.clear()
    _PTR_CHECKED[id(ptr)] = (weakref.ref(ptr), ptr._version, t, max_n)
    return max_n


def _check_packed_lattice(box, cell):
    """A packed batch takes one box [C] or cell [C, C] shared by every graph (or the [1, C] / [1, C, C] of its one
    batch row); per-graph lattices would need a graph index in every edge kernel."""
    if box is not None and torch.is_tensor(box) and box.dim() == 2 and box.shape[0] != 1:
        raise ValueError(f"ptr= takes one box [C] shared by every graph; per-graph boxes [G, C] are not supported, got "
                         f"{tuple(box.shape)}")
    if cell is not None and torch.is_tensor(cell) and cell.dim() == 3 and cell.shape[0] != 1:
        raise ValueError(f"ptr= takes one cell [C, C] shared by every graph; per-graph cells [G, C, C] are not "
                         f"supported, got {tuple(cell.shape)}")


def _packed_lattice(box, cell, dev, dtype, c):
    """The shared box [C] or cell [C, C] of a packed batch on `dev` in `dtype`, or None."""
    if cell is not None:
        return _as(cell, dev, dtype).reshape(c, c).contiguous()
    return None if box is None else _as(box, dev, dtype).reshape(c).contiguous()


_PACKED_GRID_MAX_T = (1 << 29) - 1       # 4 T bucket offsets stay an int in the grid entries


def _packed_entry(mode, t, c, k):
    """The library entry a packed select in `mode` runs: "knn" (egnn_knn_grid_select_packed: graphs large enough go on
    the kNN grid) or "radius" (egnn_radius_select_packed: on the radius grid) where the grids serve the call (C <= 3,
    k <= 256, T within the grid's int offsets), else egnn_knn_select_packed (mode None: the all-pairs select alone)."""
    if mode is None or c > 3 or k > 256 or t > _PACKED_GRID_MAX_T:
        return "egnn_knn_select_packed"
    return "egnn_radius_select_packed" if mode == "radius" else "egnn_knn_grid_select_packed"


def _in_cell_radius(r2, dtype):
    """0 < r2 < 1e5 in `dtype`, as the select compares it: the radius the radius grid serves (above, a padded pair's
    1e5 rank would count as in range)."""
    r2 = torch.tensor(float(r2), dtype=dtype).item()
    return 0.0 < r2 < 1e5


def _packed_select(x, ptr, k, m, lattice, triclinic, valid_radius, mode=None, max_n=None):
    """The packed select on staged inputs on the current device: x [1, T, C] float32 / float64, m uint8 [1, T] or
    None, lattice [C] or [C, C] (triclinic) in x's type or None -> (idx int32, ok uint8), both [1, T, k].  `mode`
    (_packed_entry) "knn": idx and ok of egnn_knn_select_packed, with the graphs of at least the kNN grid's threshold
    on that grid; "radius": its ok, and its idx in every ok = 1 slot, with the graphs of at least the radius grid's
    threshold on that grid (the callers empty the ok = 0 slots).  max_n: the largest graph's node count."""
    lib = nat.load()
    t, c = x.shape[1], x.shape[2]
    dev = x.device
    p32 = ptr.to(device=dev, dtype=torch.int32, non_blocking=True).contiguous()
    entry = _packed_entry(mode, t, c, k)
    grid = entry != "egnn_knn_select_packed"
    nb = C.c_size_t()
    nat.check(f"{entry}_workspace_bytes",
              getattr(lib, f"{entry}_workspace_bytes")(p32.numel() - 1, t, c, k, C.byref(nb)))
    stream = torch.cuda.current_stream(dev).cuda_stream
    ws = _workspace(dev, nb.value, stream)
    idx = torch.empty((1, t, k), dtype=torch.int32, device=dev)
    ok = torch.empty((1, t, k), dtype=torch.uint8, device=dev)
    name = entry + ("_triclinic" if triclinic else "")
    nat.check(name, getattr(lib, name)(_KERNEL_DTYPE[x.dtype], p32.numel() - 1, t, c, k,
                                       *((int(max_n),) if grid else ()), _ptr(p32), _ptr(x), _ptr(m),
                                       _ptr(lattice), float(valid_radius), _ptr(idx), _ptr(ok), _ptr(ws), ws.numel(),
                                       C.c_void_p(stream)))
    return idx, ok


def _packed_segments(ptr, t, dev):
    """-> (graph index [T], first node of each graph [G], node counts [G]) of a packed batch, on the device, no sync."""
    p = ptr.to(device=dev, dtype=torch.int64, non_blocking=True)
    counts = p[1:] - p[:-1]
    seg = torch.repeat_interleave(torch.arange(counts.numel(), device=dev), counts, output_size=t)
    return seg, p[:-1], counts


def _dense_packed_lists(ptr, t, max_n, dev):
    """Dense graphs of a packed batch as neighbour lists [1, T, max n_g]: slot s of a node of graph g is node
    ptr[g] + s for s < n_g, else -1.  Index arithmetic on the device, no ranking."""
    seg, start, counts = _packed_segments(ptr, t, dev)
    s = torch.arange(max_n, device=dev)
    lists = torch.where(s < counts[seg].unsqueeze(1), start[seg].unsqueeze(1) + s, -1)
    return lists.to(torch.int32).unsqueeze(0)


def edge_index_to_neighbors(edge_index, num_nodes, k=None, edge_attr=None):
    """PyG-style `edge_index` [2, E] (messages flow source j = edge_index[0] -> target i = edge_index[1], one graph)
    -> padded neighbour lists [1, N, k] for `EGNN.forward(..., neighbors=...)`; -1 marks empty slots.  Glue code:
    a stable sort by target node, nothing on the hot path.

    With `edge_attr` [E, e] (PyG's per-edge features) it returns `(neighbors, neighbor_edges)`: neighbor_edges
    [1, N, k, e] holds each edge's features in that edge's slot (same order, same truncation at k, zeros in empty
    slots), for `EGNN.forward(..., neighbors=, neighbor_edges=)`.  It is built by indexing, so gradients flow back
    to edge_attr."""
    src, dst = edge_index[0].long(), edge_index[1].long()
    order = torch.argsort(dst, stable=True)
    src, dst = src[order], dst[order]
    deg = torch.bincount(dst, minlength=num_nodes)
    kmax = int(deg.max().item()) if k is None else k
    start = torch.cumsum(deg, 0) - deg
    slot = torch.arange(src.numel(), device=src.device) - start[dst]
    out = torch.full((num_nodes, kmax), -1, dtype=torch.int32, device=src.device)
    keep = slot < kmax
    out[dst[keep], slot[keep]] = src[keep].to(torch.int32)
    if edge_attr is None:
        return out.unsqueeze(0)
    assert edge_attr.dim() == 2 and edge_attr.shape[0] == src.numel(), "edge_attr must be [E, edge_dim]"
    keep_idx = order[keep]
    slot_attr = edge_attr.new_zeros((num_nodes, kmax, edge_attr.shape[1])).index_put(
        (dst[keep], slot[keep]), edge_attr[keep_idx])
    return out.unsqueeze(0), slot_attr.unsqueeze(0)


_RADIUS_BOX_CHECKED: dict = {}


def radius_neighbors(coors, cutoff, k, *, mask=None, box=None, cell=None, return_counts=False, ptr=None):
    """Radius graph of a point cloud: for every node the (at most) `k` nearest nodes within distance `cutoff`, as int32
    neighbour lists [B, N, k] for `EGNN.forward(..., neighbors=...)`, nearest first, ties to the lower index, -1 in the
    slots left empty.  A node counts as its own neighbour (distance 0).  Computed on a cell grid (`egnn_radius_select`)
    in O(N) per graph instead of the O(N^2) ranking of the layer's kNN select, whose kept slots it equals exactly.

    `coors` float32 or float64 [B, N, C] with C <= 3, on any device (CPU tensors are staged to the current CUDA
    device; the results come back on `coors`'s device).  `cutoff` is a distance: the squared distance computed in the
    coordinates' type is compared with `float(cutoff) ** 2` cast to that type.  (The layer's `valid_radius`, as in the
    reference, is a *squared* distance.)  `k` in [1, min(32, N)] (`radius_neighbors_wide` takes up to 256).  `mask` [B, N] bool / 0-1: a padded node is never a
    neighbour and its own list is empty.  `box` [C] or [B, C]: periodic box lengths as `EGNN.forward(box=)` takes them
    (minimum-image distances; 0 or inf: the axis is not periodic).  `cell` [C, C] or [B, C, C] (C in {2, 3}), instead
    of `box`: a lower-triangular triclinic cell as `EGNN.forward(cell=)` takes it (distances of the wrapped pair
    vector; periodic axes are binned in fractional coordinates).  A node with a non-finite coordinate is never a
    neighbour and its own list is empty.

    With `return_counts=True` it returns `(neighbors, counts)`: counts int32 [B, N] is the number of nodes within the
    cutoff before the truncation at k (the node itself included), so `counts > k` shows where k cut the list short.
    Nothing synchronises with the host: the call can be captured in a CUDA graph.

    With `ptr` (a packed batch: coors [1, T, C] holding G graphs end to end, `ptr` [G+1] their offsets, as
    `EGNN.forward(ptr=)` takes them) every node is ranked against the nodes of its own graph only
    (`egnn_radius_select_packed`): on the cell grid for graphs of at least EGNN_B200_CELL_SELECT_MIN_N nodes (4096)
    and k, by the segmented all-pairs select in O(n_g^2) below: the lists equal the per-graph calls' concatenated,
    indices shifted by ptr[g], with -1 also in the slots past a graph's size (`k` up to 32 whatever the graph sizes).
    `box` / `cell` is then one lattice shared by every graph; `return_counts` is not available."""
    return _radius_graph("radius_neighbors", 32, coors, cutoff, k, mask, box, cell, return_counts, ptr)


def radius_neighbors_wide(coors, cutoff, k, *, mask=None, box=None, cell=None, return_counts=False, ptr=None):
    """`radius_neighbors` for lists of up to 256 neighbours: `k` in [1, min(256, N)], everything else the same -- the
    lists equal the all-pairs select's kept slots exactly, nearest first, ties to the lower index, -1 in the empty
    slots; `return_counts=True` also returns the in-radius counts before truncation.  For k <= 32 the result is
    `radius_neighbors`'s.  Longer lists (40-100 neighbours within a cutoff are common in condensed-phase atomistic
    systems) are kept in shared memory instead of one warp's lanes (`egnn_radius_select_wide`).  `ptr`: a packed
    batch, as `radius_neighbors` takes it (the cell grid for large graphs, `k` up to 256)."""
    return _radius_graph("radius_neighbors_wide", 256, coors, cutoff, k, mask, box, cell, return_counts, ptr)


def _check_graph_args(name, max_k, coors, k, mask, box, cell, cutoff=None, ptr=None):
    """The argument checks of the neighbour-list builders (ValueError before anything launches) -> (B, N, C).
    `cutoff` None: a builder without one (knn_neighbors).  `ptr`: a packed batch (_check_ptr), whose graphs may hold
    fewer than k nodes."""
    if not torch.is_tensor(coors) or coors.dim() != 3:
        raise ValueError(f"coors must be a [B, N, C] tensor, got {type(coors).__name__}"
                         f"{' of shape ' + str(tuple(coors.shape)) if torch.is_tensor(coors) else ''}")
    if coors.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"coors must be float32 or float64, got {coors.dtype}")
    b, n, c = coors.shape
    if b < 1 or n < 1:
        raise ValueError(f"coors must hold at least one node in at least one graph, got shape {tuple(coors.shape)}")
    if not 1 <= c <= 3:
        raise ValueError(f"{name} supports C <= 3 coordinates, got C={c}")
    k_max = max_k if ptr is not None else min(max_k, n)
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= k_max:
        raise ValueError(f"k must be an int in [1, {'' if ptr is not None else 'min('}{max_k}"
                         f"{'' if ptr is not None else ', N)'}] = [1, {k_max}], got {k!r}")
    if cutoff is not None:
        cutoff = float(cutoff)
        if not (cutoff > 0.0 and math.isfinite(cutoff)):
            raise ValueError(f"cutoff must be a finite distance > 0, got {cutoff}")
        r2 = cutoff * cutoff
        if not torch.tensor(r2, dtype=coors.dtype).item() > 0.0:
            raise ValueError(f"cutoff {cutoff} squared is 0 in {coors.dtype}")
    if mask is not None and (not torch.is_tensor(mask) or tuple(mask.shape) != (b, n)):
        raise ValueError(f"mask must be a [B, N] = [{b}, {n}] tensor, got "
                         f"{tuple(mask.shape) if torch.is_tensor(mask) else type(mask).__name__}")
    if ptr is not None:
        _check_ptr(ptr, b, n)
        _check_packed_lattice(box, cell)
    if box is not None:
        if cell is not None:
            raise ValueError("pass either box= or cell=, not both")
        _check_box(box, b, c, _RADIUS_BOX_CHECKED)
    if cell is not None:
        _check_cell(cell, b, c, _RADIUS_BOX_CHECKED)
    return b, n, c


@contextlib.contextmanager
def _grid_call(coors, k, mask, box, cell, entry):
    """The staging both cell-grid list builders share, on the compute device of `coors` (its device context held while
    the caller's block runs): coordinates, mask and the box or cell (expanded to one per graph) on that device, the
    [B, N, k] int32 output, the workspace of `entry` (a library entry point), the entry's function (its `_triclinic`
    variant under a cell) and the current stream."""
    b, n, c = coors.shape
    lib = nat.load()
    dev = _compute_device(coors)
    with _NULL_CTX if torch.cuda.current_device() == dev.index else torch.cuda.device(dev):
        if cell is not None:
            lat = _as(cell, dev, coors.dtype).expand(b, c, c).contiguous()
        else:
            lat = None if box is None else _as(box, dev, coors.dtype).expand(b, c).contiguous()
        nb = C.c_size_t()
        nat.check(f"{entry}_workspace_bytes", getattr(lib, f"{entry}_workspace_bytes")(b, n, c, k, C.byref(nb)))
        stream = torch.cuda.current_stream(dev).cuda_stream
        name = entry + ("_triclinic" if cell is not None else "")
        yield types.SimpleNamespace(dev=dev, x=_as(coors, dev, coors.dtype), m=_as_u8(mask, dev), lattice=lat,
                                    out=torch.empty((b, n, k), dtype=torch.int32, device=dev),
                                    ws=_workspace(dev, nb.value, stream), stream=stream, name=name,
                                    fn=getattr(lib, name))


def knn_neighbors(coors, k, *, mask=None, box=None, cell=None, ptr=None):
    """k-nearest-neighbour graph of a point cloud: for every node its `k` nearest nodes (itself included, distance 0),
    as int32 neighbour lists [B, N, k] for `EGNN.forward(..., neighbors=...)`, nearest first, ties to the lower index.
    The lists are those of the layer's own select (`num_nearest_neighbors=k`, no adjacency), computed on a cell grid
    (`egnn_knn_grid_select`) in O(N) per graph, with -1 in every slot the layer would not use: slots that point at a
    padded node or at a node with a non-finite coordinate, and every slot of a padded row.  Any N works, also where a
    layer with k > 32 cannot select its own lists (N > 16384).

    `coors` float32 or float64 [B, N, C] with C <= 3, on any device (CPU tensors are staged to the current CUDA
    device; the result comes back on `coors`'s device).  `k` in [1, min(256, N)].  `mask` [B, N] bool / 0-1.  `box`
    [C] or [B, C] periodic box lengths, or `cell` [C, C] or [B, C, C], as `EGNN.forward` takes them (distances of the
    wrapped pair vector).  Nothing synchronises with the host: the call can be captured in a CUDA graph.

    With `ptr` (a packed batch: coors [1, T, C] holding G graphs end to end, `ptr` [G+1] their offsets, as
    `EGNN.forward(ptr=)` takes them) every node is ranked against the nodes of its own graph only
    (`egnn_knn_grid_select_packed`): on the kNN grid for graphs of at least EGNN_B200_KNN_GRID_MIN_N nodes (8192)
    and k, by the segmented all-pairs select in O(n_g^2) below: the lists equal the per-graph calls' concatenated,
    indices shifted by ptr[g], with -1 also in the slots past a graph's size (`k` up to 256 whatever the graph sizes).
    `box` / `cell` is then one lattice shared by every graph."""
    if ptr is not None:
        return _packed_graph("knn_neighbors", 256, coors, None, k, mask, box, cell, False, ptr)
    b, n, c = _check_graph_args("knn_neighbors", 256, coors, k, mask, box, cell)
    with _grid_call(coors, k, mask, box, cell, "egnn_knn_grid_select") as g:
        x, m, out = g.x, g.m, g.out
        nat.check(g.name, g.fn(_KERNEL_DTYPE[coors.dtype], b, n, c, k, _ptr(x), _ptr(m), _ptr(g.lattice), float("inf"),
                                _ptr(out), None, _ptr(g.ws), g.ws.numel(), C.c_void_p(g.stream)))
        usable = torch.isfinite(x).all(dim=-1)                                   # [B, N]: nodes the layer uses
        if m is not None:
            usable = usable & m.bool()
        row_ok = usable if m is None else m.bool()
        keep = torch.gather(usable, 1, out.view(b, n * k).long()).view(b, n, k) & row_ok.unsqueeze(-1)
        out = out.masked_fill(~keep, -1)
    if out.device != coors.device:
        out = out.to(coors.device)
    return out


def _radius_graph(name, max_k, coors, cutoff, k, mask, box, cell, return_counts, ptr):
    if ptr is not None:
        return _packed_graph(name, max_k, coors, cutoff, k, mask, box, cell, return_counts, ptr)
    b, n, c = _check_graph_args(name, max_k, coors, k, mask, box, cell, cutoff)
    r2 = float(cutoff) * float(cutoff)
    entry = "egnn_radius_select" if max_k == 32 else "egnn_radius_select_wide"
    with _grid_call(coors, k, mask, box, cell, entry) as g:
        out = g.out
        counts = torch.empty((b, n), dtype=torch.int32, device=g.dev) if return_counts else None
        nat.check(g.name, g.fn(_KERNEL_DTYPE[coors.dtype], b, n, c, k, _ptr(g.x), _ptr(g.m), _ptr(g.lattice), r2,
                                _ptr(out), _ptr(counts), _ptr(g.ws), g.ws.numel(), C.c_void_p(g.stream)))
    if out.device != coors.device:
        out = out.to(coors.device)
        counts = None if counts is None else counts.to(coors.device)
    return (out, counts) if return_counts else out


def _packed_graph(name, max_k, coors, cutoff, k, mask, box, cell, return_counts, ptr):
    """The builders on a packed batch: the packed select (kNN or radius mode, _packed_select), then each builder's -1
    rules.  kNN (`cutoff` None): -1 in slots that point at a padded node or at a node with a non-finite coordinate, and
    in every slot of a padded row (knn_neighbors).  Radius: the kept slots are the ok = 1 slots of the select with
    valid_radius = cutoff^2 and the caller's mask -- a padded node ranks 1e5 > cutoff^2 against every node, so it is
    never kept and its own row is empty, as the radius grid leaves them; a node with a non-finite coordinate ranks inf
    or NaN against every node, itself included, and is never kept either.  Where cutoff^2 reaches 1e5 a padded node's
    coordinates are made NaN instead of passing the mask, to the same effect."""
    b, n, c = _check_graph_args(name, max_k, coors, k, mask, box, cell, cutoff, ptr)
    max_n = _check_ptr(ptr, b, n)
    if return_counts:
        raise ValueError(f"{name}: return_counts is not available with ptr=")
    dev = _compute_device(coors)
    with _NULL_CTX if torch.cuda.current_device() == dev.index else torch.cuda.device(dev):
        x, m = _as(coors, dev, coors.dtype), _as_u8(mask, dev)
        lat = _packed_lattice(box, cell, dev, coors.dtype, c)
        if cutoff is None:
            out, _ = _packed_select(x, ptr, k, m, lat, cell is not None, float("inf"), "knn", max_n)
            usable = torch.isfinite(x).all(dim=-1)                               # [1, T]: nodes the layer uses
            if m is not None:
                usable = usable & m.bool()
            row_ok = usable if m is None else m.bool()
            filled = out >= 0
            keep = filled & torch.gather(usable, 1, out.clamp_min(0).view(b, n * k).long()).view(b, n, k)
            keep &= row_ok.unsqueeze(-1)
        else:
            r2 = float(cutoff) * float(cutoff)
            if m is not None and not _in_cell_radius(r2, coors.dtype):
                x, m = x.masked_fill(~m.bool().unsqueeze(-1), float("nan")), None
            out, ok = _packed_select(x, ptr, k, m, lat, cell is not None, r2, "radius", max_n)
            keep = ok.bool()
        out = out.masked_fill(~keep, -1)
    return out if out.device == coors.device else out.to(coors.device)


# ----------------------------------------------------------------------------- global attention


class _Attention(nn.Module):
    """Parameter holder (+ autograd path) of the multi-head softmax attention inside GlobalLinearAttention
    (reference egnn_pytorch.py:81-110): `to_q`, `to_kv` without bias, `to_out` with bias."""

    def __init__(self, dim, heads=8, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim, inner * 2, bias=False)
        self.to_out = nn.Linear(inner, dim)

    def forward(self, x, context, mask=None):
        """Training path (PyTorch autograd).  Masked keys get the most negative finite score BEFORE the softmax, like the
        reference (:101-104), so a fully masked graph attends uniformly instead of producing NaN."""
        h = self.heads
        q = self.to_q(x)
        k, v = self.to_kv(context).chunk(2, dim=-1)
        split = lambda t: t.unflatten(-1, (h, -1)).transpose(1, 2)
        q, k, v = split(q), split(k), split(v)
        dots = (q @ k.transpose(-1, -2)) * self.dim_head ** -0.5
        if mask is not None:
            dots = dots.masked_fill(~mask[:, None, None, :].to(torch.bool), -torch.finfo(dots.dtype).max)
        out = dots.softmax(dim=-1) @ v
        return self.to_out(out.transpose(1, 2).flatten(-2))


class GlobalLinearAttention(nn.Module):
    """Induced-set attention between the nodes and a few global tokens (reference egnn_pytorch.py:112-144).

    Inference (no autograd recording): ONE call of `egnn_global_attn_forward` (csrc/global_attn.cu) on staged fp32 / fp64
    copies of the parameters -- the module itself is never moved.  When a gradient is required, or there are more than 32
    global tokens, the same arithmetic runs through PyTorch (the hand-written backward of SURVEY.md section 8(f) covers
    the EGNN layers only).  A size-1 batch of `x`, `queries` or `mask` is broadcast, as in the reference."""

    def __init__(self, *, dim, heads=8, dim_head=64):
        super().__init__()
        self.dim, self.heads, self.dim_head = dim, heads, dim_head
        self.norm_seq = nn.LayerNorm(dim)
        self.norm_queries = nn.LayerNorm(dim)
        self.attn1 = _Attention(dim, heads, dim_head)
        self.attn2 = _Attention(dim, heads, dim_head)
        self.ff = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, dim * 4), nn.GELU(), nn.Linear(dim * 4, dim))
        self._stage = {}

    def _forward_autograd(self, x, queries, mask=None):
        nx, nq = self.norm_seq(x), self.norm_queries(queries)
        induced = self.attn1(nq, nx, mask=mask)
        x = self.attn2(nx, induced) + x
        queries = induced + queries
        return self.ff(x) + x, queries

    def _staged(self, device, dtype):
        """-> (sig, tensors, weights struct, built): the staged parameters for (device, dtype) and their stream order."""
        named = [(k, p) for k, p in self.named_parameters() if k in nat.GA_STATE_KEY_TO_FIELD]
        sig = tuple((p.data_ptr(), p._version) for _, p in named)
        st = self._stage.get((device, dtype))
        if st is None or st[0] != sig:
            with torch.no_grad():
                tensors = {nat.GA_STATE_KEY_TO_FIELD[k]: p.detach().to(device=device, dtype=dtype).contiguous() for k, p in named}
            w = nat.GlobalAttnWeights(**{f: t.data_ptr() for f, t in tensors.items()})
            st = (sig, tensors, w, _Built(torch.cuda.current_stream(device), list(tensors.values())))
            self._stage[(device, dtype)] = st
        return st

    def invalidate_cache(self):
        self._stage = {}

    def _batch(self, x, queries, mask):
        """Shape check -> the common batch B.  x [Bx, N, dim], queries [Bq, T, dim], mask [Bm, N]; each of Bx, Bq, Bm is 1
        or B, as the reference's einsum and masked_fill broadcast a size-1 batch."""
        def shape(t):
            return tuple(t.shape) if torch.is_tensor(t) else type(t).__name__
        if not (torch.is_tensor(x) and x.dim() == 3 and x.shape[2] == self.dim):
            raise ValueError(f"x must be [B, N, dim={self.dim}], got {shape(x)}")
        if not (torch.is_tensor(queries) and queries.dim() == 3 and queries.shape[2] == self.dim):
            raise ValueError(f"queries must be [B, T, dim={self.dim}], got {shape(queries)}")
        batches = [x.shape[0], queries.shape[0]]
        if mask is not None:
            if not (torch.is_tensor(mask) and mask.dim() == 2 and mask.shape[1] == x.shape[1]):
                raise ValueError(f"mask must be [B, N={x.shape[1]}], got {shape(mask)}")
            batches.append(mask.shape[0])
        b = max(batches)
        if any(v not in (1, b) for v in batches):
            raise ValueError(f"batch sizes of x, queries and mask must each be 1 or the same B, got {batches}")
        return b

    def forward(self, x, queries, mask=None):
        b = self._batch(x, queries, mask)
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or queries.requires_grad or
                                                  any(p.requires_grad for p in self.parameters()))
        # T > 32: ga_attn2_kernel keeps a node's T scores in registers, so more tokens take the autograd path's arithmetic
        if needs_grad or queries.shape[1] > 32:
            dev = x.device
            if any(p.device != dev for p in self.parameters()):
                raise RuntimeError("training GlobalLinearAttention, or running it with more than 32 global tokens, needs "
                                   "the module on the device of its inputs")
            return self._forward_autograd(x, queries, mask)
        lib = nat.load()
        dev = _compute_device(x)
        kdt = torch.float64 if x.dtype == torch.float64 else torch.float32
        cs = torch.cuda.current_stream(dev)
        _, _, w, built = self._staged(dev, kdt)
        if built.stream != cs.cuda_stream:
            built.use_on(cs)
        n, d, t = x.shape[1], x.shape[2], queries.shape[1]
        x, queries = x.expand(b, -1, -1), queries.expand(b, -1, -1)
        mask = None if mask is None else mask.expand(b, -1)
        x_in, q_in, m_in = _as(x, dev, kdt), _as(queries, dev, kdt), _as_u8(mask, dev)
        x_out, q_out = torch.empty_like(x_in), torch.empty_like(q_in)
        desc = nat.GlobalAttnDesc(abi_version=nat.ABI_VERSION, dtype=_KERNEL_DTYPE[kdt], B=b, N=n, T=t, dim=d, heads=self.heads,
                                  dim_head=self.dim_head)
        nb = C.c_size_t()
        nat.check("egnn_global_attn_workspace_bytes", lib.egnn_global_attn_workspace_bytes(C.byref(desc), C.byref(nb)))
        io = nat.GlobalAttnIO(x=x_in.data_ptr(), queries=q_in.data_ptr(), mask=None if m_in is None else m_in.data_ptr(),
                              x_out=x_out.data_ptr(), queries_out=q_out.data_ptr())
        with torch.cuda.device(dev):
            ws = _workspace(dev, nb.value)
            nat.check("egnn_global_attn_forward",
                      lib.egnn_global_attn_forward(C.byref(desc), C.byref(w), C.byref(io), _ptr(ws), ws.numel(),
                                                   C.c_void_p(cs.cuda_stream)))
        return x_out.to(device=x.device, dtype=x.dtype), q_out.to(device=queries.device, dtype=queries.dtype)


# ----------------------------------------------------------------------------- the network


def _adj_cache_key(adj_mat, b, num_adj_degrees):
    """What EGNN_Network's expanded adjacency depends on: the storage and its version, and the view of it -- `A.t()` or a
    dtype view shares A's pointer, version counter and shape but holds another matrix."""
    return (adj_mat.data_ptr(), adj_mat._version, tuple(adj_mat.shape), adj_mat.stride(), adj_mat.dtype, b,
            num_adj_degrees)


class EGNN_Network(nn.Module):
    """Drop-in for `egnn_pytorch.EGNN_Network` (reference egnn_pytorch.py:343-454).

    Differences in mechanism, not in results: the N-th degree adjacency is expanded on bit-packed
    rows by `egnn_adj_expand` instead of dense `A @ A` (:425), and the adjacency-degree embedding
    is never materialised as a [B,N,N,adj_dim] tensor (:430-432) -- layers receive the uint8 degree
    labels and fold `adj_emb.weight` into a [num_degrees+1, H] table."""

    def __init__(self, *, depth, dim, num_tokens=None, num_edge_tokens=None, num_positions=None, edge_dim=0,
                 num_adj_degrees=None, adj_dim=0, global_linear_attn_every=0, global_linear_attn_heads=8,
                 global_linear_attn_dim_head=64, num_global_tokens=4, **kwargs):
        super().__init__()
        assert not (exists(num_adj_degrees) and num_adj_degrees < 1), "make sure adjacent degrees is greater than 1"
        self.num_positions = num_positions
        self.token_emb = nn.Embedding(num_tokens, dim) if exists(num_tokens) else None
        self.pos_emb = nn.Embedding(num_positions, dim) if exists(num_positions) else None
        self.edge_emb = nn.Embedding(num_edge_tokens, edge_dim) if exists(num_edge_tokens) else None
        self.has_edges = edge_dim > 0
        self.num_adj_degrees = num_adj_degrees
        self.adj_emb = nn.Embedding(num_adj_degrees + 1, adj_dim) if exists(num_adj_degrees) and adj_dim > 0 else None
        edge_dim = edge_dim if self.has_edges else 0
        adj_dim = adj_dim if exists(num_adj_degrees) else 0
        has_global_attn = global_linear_attn_every > 0
        self.global_tokens = nn.Parameter(torch.randn(num_global_tokens, dim)) if has_global_attn else None
        self.layers = nn.ModuleList()
        for ind in range(depth):
            is_global = has_global_attn and (ind % global_linear_attn_every) == 0
            self.layers.append(nn.ModuleList([
                GlobalLinearAttention(dim=dim, heads=global_linear_attn_heads,
                                      dim_head=global_linear_attn_dim_head) if is_global else None,
                EGNN(dim=dim, edge_dim=edge_dim + adj_dim, norm_feats=True, **kwargs),
            ]))

    def forward(self, feats, coors, adj_mat=None, edges=None, mask=None, return_coor_changes=False, *, box=None,
                cell=None, lattice_grad=False, ptr=None):
        """`box` (additive, keyword-only): periodic box lengths [C] or [B, C], passed to every layer (EGNN.forward).
        `cell` (additive, keyword-only, instead of `box`): a lower-triangular triclinic cell [C, C] or [B, C, C], passed
        to every layer (EGNN.forward).  `lattice_grad` (additive, keyword-only): passed to every layer, so a box / cell
        that requires grad gets the sum of the layers' lattice gradients, through the chained coordinates too.
        `ptr` (additive, keyword-only): a packed batch of variable-size graphs, feats [1, T] (tokens) or [1, T, dim] and
        coors [1, T, C] with graph g on nodes ptr[g] .. ptr[g+1]-1 (EGNN.forward).  Every layer ranks each graph's
        nodes from its own input coordinates; positions restart at every graph (node i of graph g is at position
        i - ptr[g], and the largest graph must fit num_positions).  Adjacency, dense edges and global linear
        attention are not available with it (ValueError)."""
        _check_lattice(box, cell, feats.shape[0], coors.shape[-1], self.__dict__, lattice_grad)
        if ptr is not None:
            if adj_mat is not None or exists(self.num_adj_degrees) or exists(edges) or exists(self.global_tokens):
                raise ValueError("ptr= (a packed batch) cannot be combined with adj_mat / num_adj_degrees, dense edges or "
                                 "global linear attention")
            max_n = _check_ptr(ptr, feats.shape[0], feats.shape[1])
        lib = nat.load()
        out_dev = coors.device
        dev = _compute_device(coors)
        b = feats.shape[0]
        feats, coors = feats.to(dev), coors.to(dev)
        adj_mat = None if adj_mat is None else adj_mat.to(dev)
        edges = None if edges is None else edges.to(dev)
        mask = None if mask is None else mask.to(dev)

        def staged(emb):
            return emb.weight if emb.weight.device == dev else emb.weight.to(dev)

        if exists(self.pos_emb):
            n = feats.shape[1] if ptr is None else max_n
            assert n <= self.num_positions, \
                f"given sequence length {n} must be less than the number of positions {self.num_positions} set at init"
        emb_grad = torch.is_grad_enabled() and any(e is not None and e.weight.requires_grad for e in (self.token_emb, self.pos_emb))
        if exists(self.token_emb) and not emb_grad and self.token_emb.weight.dtype in _KERNEL_DTYPE and ptr is None:
            # token + positional embedding in ONE launch (egnn_embed_nodes) instead of embedding, arange, embedding, add
            tw = staged(self.token_emb)
            pw = staged(self.pos_emb) if exists(self.pos_emb) else None
            tok = feats.to(torch.int64).contiguous()
            n = tok.shape[1]
            feats = torch.empty((b, n, tw.shape[1]), dtype=tw.dtype, device=dev)
            with (_NULL_CTX if torch.cuda.current_device() == dev.index else torch.cuda.device(dev)):
                nat.check("egnn_embed_nodes", lib.egnn_embed_nodes(
                    _KERNEL_DTYPE[tw.dtype], b, n, tw.shape[1], tw.shape[0], _ptr(tok), _ptr(tw), _ptr(pw), _ptr(feats),
                    C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        else:                                        # training through the embedding tables: PyTorch autograd
            if exists(self.token_emb):
                feats = F.embedding(feats, staged(self.token_emb))                   # reference :401-402
            if exists(self.pos_emb) and ptr is not None:          # positions restart at every graph of a packed batch
                seg, start, _ = _packed_segments(ptr, feats.shape[1], dev)
                feats = feats + staged(self.pos_emb)[torch.arange(feats.shape[1], device=dev) - start[seg]].unsqueeze(0)
            elif exists(self.pos_emb):
                feats = feats + staged(self.pos_emb)[:feats.shape[1]].unsqueeze(0)   # :404-408
        if exists(edges) and exists(self.edge_emb):
            edges = F.embedding(edges, staged(self.edge_emb))                        # :410-411

        labels = label_emb = k_hint = nbr_lists = None
        if exists(self.num_adj_degrees):
            assert exists(adj_mat), "adjacency matrix must be passed in (keyword argument adj_mat)"
            # the expansion depends on the adjacency only: cached per view of a storage version, which also keeps the
            # reference's host sync (:249) out of repeated calls and makes the forward CUDA-graph capturable
            akey = _adj_cache_key(adj_mat, b, self.num_adj_degrees)
            cached = self.__dict__.get("_adj_cache")
            cs = torch.cuda.current_stream(dev)
            if cached is not None and cached[0] == akey:
                if cached[6].stream != cs.cuda_stream:
                    cached[6].use_on(cs)
            else:
                n = adj_mat.shape[-1]
                adj_in = adj_mat.ne(0).to(torch.uint8).contiguous()
                adj_out = torch.empty((b, n, n), dtype=torch.uint8, device=dev)
                lab = torch.empty((b, n, n), dtype=torch.uint8, device=dev)
                max_sum = torch.zeros(1, dtype=torch.int32, device=dev)
                nb = C.c_size_t()
                nat.check("egnn_adj_workspace_bytes", lib.egnn_adj_workspace_bytes(b, n, C.byref(nb)))
                with torch.cuda.device(dev):
                    ws = _workspace(dev, nb.value)
                    nat.check("egnn_adj_expand", lib.egnn_adj_expand(
                        b, n, self.num_adj_degrees, _ptr(adj_in), 1 if adj_in.dim() == 3 else 0, _ptr(adj_out), _ptr(lab),
                        _ptr(max_sum), _ptr(ws), ws.numel(), C.c_void_p(cs.cuda_stream)))
                kmax = int(max_sum.item()) if self.layers[0][1].only_sparse_neighbors else None   # the reference's sync at :249
                # only_sparse_neighbors with a node mask: the surviving slots of every layer's top-k are the node and its
                # adjacent nodes (valid_radius = 0, :250, :296) -- lists that depend on the adjacency only.  Built once
                # here (egnn_adj_neighbors) and handed to every layer instead of one adjacency scan per layer.
                lists = None
                if kmax is not None and 0 < kmax <= n and os.environ.get("EGNN_B200_NO_LIST_CACHE") != "1":
                    lists = torch.empty((b, n, kmax), dtype=torch.int32, device=dev)
                    with torch.cuda.device(dev):
                        nat.check("egnn_adj_neighbors", lib.egnn_adj_neighbors(
                            b, n, kmax, _ptr(adj_out), 1, _ptr(lists), None, C.c_void_p(cs.cuda_stream)))
                built = _Built(cs, [adj_out, lab] + ([] if lists is None else [lists]))
                cached = (akey, adj_out, lab, kmax, adj_mat, lists, built)   # adj_mat kept alive so the key cannot be recycled
                self.__dict__["_adj_cache"] = cached
            _, adj_out, lab, k_hint, _, nbr_lists, _ = cached
            adj_mat = adj_out                                                        # layers see the expanded matrix (:428, :448)
            if exists(self.adj_emb):
                labels, label_emb = lab, self.adj_emb.weight

        global_tokens = None
        if exists(self.global_tokens):
            global_tokens = self.global_tokens.to(dev).unsqueeze(0).expand(b, -1, -1)

        coor_changes = [coors]
        for global_attn, egnn in self.layers:
            if exists(global_attn):
                feats, global_tokens = global_attn(feats, global_tokens, mask=mask)
            feats, coors = egnn(feats, coors, edges, mask, adj_mat, _edge_labels=labels, _label_emb=label_emb,
                                _k_hint=k_hint, neighbors=nbr_lists if exists(mask) else None, box=box, cell=cell,
                                lattice_grad=lattice_grad, ptr=ptr)
            coor_changes.append(coors)

        if out_dev != dev:
            feats, coors = feats.to(out_dev), coors.to(out_dev)
        if return_coor_changes:
            return feats, coors, [c.to(out_dev) for c in coor_changes]
        return feats, coors

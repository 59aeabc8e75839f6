"""Multi-GPU use of the layer (SURVEY.md section 8(e)).  One process per GPU, torch.distributed for
the plumbing.

* Batches of independent graphs shard over ranks with NO data-path collective
  (`batch_shard`, `batch_sharded_call`); outputs are gathered only if the caller asks.
* One huge graph: contiguous blocks of i-rows per rank.  Every rank needs all coordinates and all
  node features (for the per-node B_j table), so each layer starts with ONE all-gather of
  [coors | feats] and then evaluates only its own rows (`row_sharded_layer_call`); top-k, masks and
  both j-reductions are row-local, so nothing is reduced across ranks.

* Training on batch shards: every rank differentiates the loss of its own graphs; the parameter gradients are
  the only thing exchanged -- `allreduce_gradients` sums them in a few flat buckets (one collective per
  bucket: the whole EGNN(512) layer is 12.8 MB in fp32, i.e. one launch-latency-bound all-reduce over NVLink).
* Training on row shards of one graph: the gather is differentiable.  Its backward all-reduces (sums) the
  full-size gradient of [coors | feats] and keeps this rank's rows; each rank's layer backward covers its own
  row block only (EGNN_FLAG_ROW_PARTIAL_GRADS, per-pair memory ~ rows / world), so the parameter gradients are
  partial sums that the same `allreduce_gradients` completes.

The compute callable is injected, so the partition/exchange logic is testable on CPU with gloo
(tests/test_multi_rank_cpu.py drives it with the oracle); on the GPU box it is the CUDA module.

On H100s the all-gather of the row-sharded graph is NOT a host-driven collective: `PeerComm` wraps the library's
peer-memory communicator (`egnn_comm_*`, csrc/peer_comm.cu) -- one kernel per rank pushes the rank's rows into every
peer's buffer with P2P stores over NVLink and waits on device-side epoch flags, enqueued on the layer's own stream
(`row_sharded_layer_peer`).  torch.distributed is only used once, to exchange the 64-byte IPC handles.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.distributed as dist


def shard_range(total: int, rank: int, world: int):
    """Contiguous, balanced [begin, end) of `total` units for `rank` (first ranks get the remainder)."""
    base, rem = divmod(total, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def batch_shard(tensors: dict, rank: int, world: int, batch: int):
    """Slice every tensor whose leading dimension is the batch; 2-D adjacency etc. pass through."""
    b0, b1 = shard_range(batch, rank, world)
    out = {}
    for k, v in tensors.items():
        if torch.is_tensor(v) and v.dim() >= 1 and v.shape[0] == batch and not (k == "adj_mat" and v.dim() == 2):
            out[k] = v[b0:b1]
        else:
            out[k] = v
    return out, (b0, b1)


def _all_gather_var(x: torch.Tensor, sizes, group=None):
    """all_gather of per-rank blocks with different leading sizes (pads to the maximum)."""
    world = dist.get_world_size(group)
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    pad[: x.shape[0]] = x
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    return torch.cat([b[:s] for b, s in zip(bufs, sizes)], dim=0)


def batch_sharded_call(fn, tensors: dict, batch: int, gather: bool = True, group=None):
    """Run `fn(**shard)` on this rank's graphs; optionally all-gather the (feats, coors) outputs."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    if gather and batch < world:
        # checked identically on every rank BEFORE any collective: a rank with an empty shard would have nothing to
        # contribute to the all-gather and the others would wait for it forever
        raise ValueError(f"batch_sharded_call(gather=True) needs at least one graph per rank (batch={batch}, world={world}); "
                         f"use a smaller process group or gather=False")
    shard, (b0, b1) = batch_shard(tensors, rank, world, batch)
    outs = fn(**shard) if b1 > b0 else None
    if not gather:
        return outs
    sizes = [shard_range(batch, r, world)[1] - shard_range(batch, r, world)[0] for r in range(world)]
    return tuple(_all_gather_var(o, sizes, group) for o in outs)


class _GatherRows(torch.autograd.Function):
    """All-gather of the per-rank row blocks along dim 0.  Every rank's rows feed every rank's layer (as neighbours j),
    so the gradient of a rank's block is the SUM over ranks of the gradient of the gathered array, taken at the block's
    rows: one all-reduce of the full-size gradient, then a slice (gloo has no reduce-scatter; the payload is only
    N x (C + dim)).  Every rank must run its backward: the all-reduce is a collective."""

    @staticmethod
    def forward(ctx, local, sizes, rank, group):
        ctx.sizes, ctx.rank, ctx.group = sizes, rank, group
        return _all_gather_var(local, sizes, group)

    @staticmethod
    def backward(ctx, g):
        g = g.clone(memory_format=torch.contiguous_format)
        dist.all_reduce(g, op=dist.ReduceOp.SUM, group=ctx.group)
        r0 = sum(ctx.sizes[:ctx.rank])
        return g[r0:r0 + ctx.sizes[ctx.rank]], None, None, None


def row_sharded_layer_call(layer_fn, feats_local, coors_local, n_total: int, group=None, **kw):
    """One layer of a row-sharded single graph.

    feats_local [B, R_rank, dim], coors_local [B, R_rank, C] hold this rank's node block.  The single
    exchange step all-gathers both along the node axis; `layer_fn(feats_all, coors_all, rows=(r0, r1), **kw)`
    must return full-size outputs of which only rows r0:r1 are meaningful.  Returns the local blocks.

    Training: the call is differentiable.  `layer_fn` must differentiate as the function it returns (an `EGNN` called
    with `_rows=` does), and the gather's backward sums the gradient of the gathered array over the ranks and hands each
    rank its own rows, so gradients reach `feats_local` / `coors_local` and layers chain.  After `loss.backward()` every
    rank holds its block's PARTIAL sum of each parameter gradient: `allreduce_gradients(params)` (sum, not average)
    completes them.  With dropout, every rank must draw the same per-call seed (e.g. the same `torch.manual_seed` on
    every rank): the masks are keyed on global pair indices, so the sharded step then equals the single-GPU step."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    sizes = [shard_range(n_total, r, world)[1] - shard_range(n_total, r, world)[0] for r in range(world)]
    r0, r1 = shard_range(n_total, rank, world)
    # one payload: [coors | feats] along the channel axis, node axis first for the gather
    wide = torch.promote_types(coors_local.dtype, feats_local.dtype)      # bf16 feats ride in fp32: exact
    payload = torch.cat([coors_local.to(wide), feats_local.to(wide)], dim=-1).transpose(0, 1).contiguous()
    full = _GatherRows.apply(payload, sizes, rank, group).transpose(0, 1)
    c = coors_local.shape[-1]
    coors_all = full[..., :c].to(coors_local.dtype).contiguous()
    feats_all = full[..., c:].to(feats_local.dtype).contiguous()
    f_out, x_out = layer_fn(feats_all, coors_all, rows=(r0, r1), **kw)
    return f_out[:, r0:r1], x_out[:, r0:r1]


def allreduce_gradients(params, group=None, average: bool = False, bucket_bytes: int = 64 << 20):
    """Sum (or average) `.grad` of the given parameters over the ranks, in place.

    Gradients are packed into flat buckets of at most `bucket_bytes` per dtype so that a layer costs one collective
    instead of one per tensor.  Parameters whose `.grad` is None on this rank (e.g. a rank with an empty shard)
    contribute zeros -- every rank must pass the same parameter list in the same order."""
    world = dist.get_world_size(group)
    params = [p for p in params if p.requires_grad]
    by_dtype = {}
    for p in params:
        by_dtype.setdefault((p.dtype, p.device), []).append(p)
    for (dtype, device), plist in by_dtype.items():
        bucket, size = [], 0
        buckets = []
        for p in plist:
            nbytes = p.numel() * p.element_size()
            if bucket and size + nbytes > bucket_bytes:
                buckets.append(bucket)
                bucket, size = [], 0
            bucket.append(p)
            size += nbytes
        if bucket:
            buckets.append(bucket)
        for bucket in buckets:
            flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in bucket])
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
            if average:
                flat /= world
            off = 0
            for p in bucket:
                g = flat[off:off + p.numel()].view_as(p)
                if p.grad is None:
                    p.grad = g.clone()
                else:
                    p.grad.copy_(g)
                off += p.numel()


# ----------------------------------------------------------------------------- peer-memory all-gather (NVLink)


class _DeviceBytes:
    """Raw device memory as a __cuda_array_interface__ object (the gather buffer is owned by the library)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(ptr, False), version=2)


class PeerComm:
    """One per process / GPU.  `payload_bytes` = size of the gathered [coors | feats] arrays of one call."""

    def __init__(self, payload_bytes: int, group=None):
        from . import _native as nat
        self.nat, self.lib = nat, nat.load()
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.payload_bytes = int(payload_bytes)
        self.handle = C.c_void_p()
        ipc = (C.c_ubyte * 64)()
        nat.check("egnn_comm_create", self.lib.egnn_comm_create(self.world, self.rank, self.payload_bytes, C.byref(self.handle), ipc))
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(ipc), group=group)
        blob = (C.c_ubyte * (64 * self.world)).from_buffer_copy(b"".join(handles))
        nat.check("egnn_comm_connect", self.lib.egnn_comm_connect(self.handle, blob))
        dist.barrier(group)                       # every rank has mapped every buffer before the first push

    def allgather(self, segments, device):
        """segments: [(tensor (contiguous, this rank's rows), dst_byte_offset)].  Returns a uint8 tensor viewing the
        complete gathered buffer of this call (valid until the call after next)."""
        n = len(segments)
        src = (C.c_void_p * n)(*[t.data_ptr() for t, _ in segments])
        off = (C.c_size_t * n)(*[int(o) for _, o in segments])
        nb = (C.c_size_t * n)(*[t.numel() * t.element_size() for t, _ in segments])
        out = C.c_void_p()
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        self.nat.check("egnn_comm_allgather", self.lib.egnn_comm_allgather(self.handle, n, src, off, nb, C.byref(out), stream))
        return torch.as_tensor(_DeviceBytes(out.value, self.payload_bytes), device=device)

    def status(self):
        st = C.c_int32()
        self.nat.check("egnn_comm_status", self.lib.egnn_comm_status(self.handle, C.byref(st)))
        return st.value

    def close(self):
        if self.handle:
            self.lib.egnn_comm_destroy(self.handle)
            self.handle = None


def row_payload_layout(n_total: int, c: int, dim: int, feat_bytes: int, batch: int = 1):
    """Byte layout of one gathered call: coors [B,N,C] fp32 at 0, feats [B,N,dim] at a 256-aligned offset."""
    coors_bytes = batch * n_total * c * 4
    feats_off = (coors_bytes + 255) // 256 * 256
    return feats_off, feats_off + batch * n_total * dim * feat_bytes


def _peer_gather(comm: PeerComm, feats_local, coors_local, n_total: int):
    """-> (feats_all, coors_all): views of the communicator's gather buffer, valid until the call after next."""
    dev = feats_local.device
    b, _, dim = feats_local.shape
    c = coors_local.shape[-1]
    r0, _ = shard_range(n_total, comm.rank, comm.world)
    feats_off, total = row_payload_layout(n_total, c, dim, feats_local.element_size(), b)
    assert total <= comm.payload_bytes, "PeerComm payload too small for this graph"
    coors_local = coors_local.contiguous()
    feats_local = feats_local.contiguous()
    segs = []
    for g in range(b):            # rows of one graph are contiguous in both the local block and the gathered array
        segs.append((coors_local[g], (g * n_total + r0) * c * 4))
        segs.append((feats_local[g], feats_off + (g * n_total + r0) * dim * feats_local.element_size()))
    buf = comm.allgather(segs, dev)
    coors_all = buf[:b * n_total * c * 4].view(torch.float32).view(b, n_total, c)
    feats_all = buf[feats_off:total].view(feats_local.dtype).view(b, n_total, dim)
    return feats_all, coors_all


class _PeerGatherRows(torch.autograd.Function):
    """The peer-memory all-gather under autograd.  The gathered arrays are copied out of the communicator's buffer into
    tensors torch owns: the layer saves its inputs for backward, and the buffer is rewritten by the call after next --
    raw memory whose reuse the saved-tensor version check cannot see.  Backward as `_GatherRows`: one all-reduce (sum) of
    the full-size gradients over `comm.group`, then this rank's rows."""

    @staticmethod
    def forward(ctx, feats_local, coors_local, comm, n_total):
        ctx.group, ctx.rows = comm.group, shard_range(n_total, comm.rank, comm.world)
        feats_all, coors_all = _peer_gather(comm, feats_local, coors_local, n_total)
        return feats_all.clone(), coors_all.clone()

    @staticmethod
    def backward(ctx, g_f, g_x):
        wide = torch.promote_types(g_x.dtype, g_f.dtype)
        flat = torch.cat([g_x.to(wide).reshape(-1), g_f.to(wide).reshape(-1)])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=ctx.group)
        g_x_all = flat[:g_x.numel()].view(g_x.shape)
        g_f_all = flat[g_x.numel():].view(g_f.shape)
        r0, r1 = ctx.rows
        return g_f_all[:, r0:r1].to(g_f.dtype), g_x_all[:, r0:r1].to(g_x.dtype), None, None


def row_sharded_layer_peer(comm: PeerComm, layer, feats_local, coors_local, n_total: int, **kw):
    """One layer of a row-sharded single graph with the peer-memory all-gather.

    feats_local [B, R_rank, dim] (module dtype), coors_local [B, R_rank, C] float32: this rank's node block (rows
    `shard_range(n_total, rank, world)`).  Pushes both into every rank's gather buffer (one kernel, NVLink), then runs
    `layer(feats_all, coors_all, _rows=(r0, r1), **kw)` on the gathered arrays.  Returns the local output blocks.

    Under `torch.no_grad()` the layer reads the gathered arrays in place.  With grad mode on they are copied into tensors
    torch owns (the layer may save them for backward), and the call differentiates like `row_sharded_layer_call`: gradients
    reach `feats_local` / `coors_local`, and `allreduce_gradients` (sum) completes the parameter gradients."""
    r0, r1 = shard_range(n_total, comm.rank, comm.world)
    coors_local = coors_local.float()
    # under grad the layer may save its inputs whatever `layer` is (a module, a lambda around one, ...): always copy
    if torch.is_grad_enabled():
        feats_all, coors_all = _PeerGatherRows.apply(feats_local, coors_local, comm, n_total)
    else:
        feats_all, coors_all = _peer_gather(comm, feats_local, coors_local, n_total)
    f_out, x_out = layer(feats_all, coors_all, _rows=(r0, r1), **kw)
    return f_out[:, r0:r1], x_out[:, r0:r1]


def row_sharded_benchmark(world: int, rank: int, dev, n_total: int = 8192, dim: int = 512, iters: int = 5):
    """`bench.py`'s strong-scaling probe (world > 1): ONE dense graph, EGNN(dim) bf16, N = n_total, i-rows split over
    the ranks, one peer-memory all-gather of [coors | feats] per layer call.  Time = CUDA events around
    (all-gather + layer) per iteration, max over ranks; the single-GPU time of the same graph is measured on rank 0
    in the same process; parity = max |row-sharded - single-rank| over all rows (bf16 feats, fp32 coors)."""
    from .egnn import EGNN
    torch.manual_seed(0)                                  # identical weights and inputs on every rank
    layer = EGNN(dim=dim).bfloat16().to(dev).eval()
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(1, n_total, dim, generator=g).to(dev, torch.bfloat16)
    coors = torch.randn(1, n_total, 3, generator=g).to(dev)
    r0, r1 = shard_range(n_total, rank, world)
    _, payload = row_payload_layout(n_total, 3, dim, 2)
    comm = PeerComm(payload)
    f_loc, x_loc = feats[:, r0:r1].contiguous(), coors[:, r0:r1].contiguous()

    def sharded():
        return row_sharded_layer_peer(comm, layer, f_loc, x_loc, n_total)

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize(dev)
        dist.barrier()
        torch.cuda.synchronize(dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            out = fn()
        b.record()
        torch.cuda.synchronize(dev)
        return a.elapsed_time(b) / n, out

    with torch.no_grad():
        ms, (f_sh, x_sh) = timed(sharded, iters)
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
        # the same graph on ONE GPU (every rank runs it, so the parity check needs no broadcast; rank 0's time is reported)
        ms1, (f_full, x_full) = timed(lambda: layer(feats, coors), 3)
        err = torch.tensor([float((f_sh.float() - f_full[:, r0:r1].float()).abs().max()),
                            float((x_sh - x_full[:, r0:r1]).abs().max())], dtype=torch.float64, device=dev)
        dist.all_reduce(err, op=dist.ReduceOp.MAX)
        t1 = torch.tensor([ms1], dtype=torch.float64, device=dev)
        dist.broadcast(t1, src=0)
        ms1 = float(t1.item())
    status = comm.status()
    comm.close()
    pairs = n_total * n_total
    return dict(workload=f"EGNN(dim={dim}) dense all-pairs, ONE graph N={n_total}, bf16, i-rows sharded x{world}",
                ms=ms, pairs_per_s=pairs / ms * 1e3, ms_1gpu=ms1, speedup_vs_1gpu=ms1 / ms, efficiency_vs_1gpu=ms1 / (world * ms),
                parity_max_err_vs_single_rank=dict(feats=float(err[0]), coors=float(err[1])),
                collective="peer-memory all-gather: one push kernel per rank, P2P stores over NVLink + device-side epoch flags "
                           "(egnn_comm_allgather, csrc/peer_comm.cu), on the layer's stream; no NCCL, no host sync",
                bytes_received_per_rank=int((n_total - (r1 - r0)) * (dim * 2 + 12)), comm_status=status,
                kernel_path=layer.last_path, scaling="strong", iters=iters)

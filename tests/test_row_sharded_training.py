"""Training of row blocks (EGNN_FLAG_ROW_PARTIAL_GRADS) and of row-sharded single graphs (parallel.py).

A row block [r0, r1) of a layer returns the gradient of sum_{b, i in block} <g_out[b,i], out[b,i]>: its own rows' terms
and the neighbour-side terms of every row.  The reference for one block is the numpy backward oracle with the cotangents
zeroed outside the block; the blocks of a partition must sum to the whole layer's gradient."""
import functools
import math
import os
import ctypes as C

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import cases
import util
from oracle import egnn_oracle as O
from oracle import egnn_oracle_grad as G
from util import nat  # noqa: F401  (module-scoped fixture)

# dense N = 97 with Hp = 152: blocks cross the 32-row tiles and the 128-channel tiles of the dense bwd2
N97 = dict(kind="layer", cfg=dict(dim=36, edge_dim=2, norm_feats=True), B=1, N=97, seed=70, init="xavier", mask="padded")
BLOCK_CASES = ["dense_everything", "dense_mask_padded", "dense_mdim32", "dense_fourier", "dense_no_feats", "dense_no_coors",
               "knn_edges_mask", "knn_mean_fourier", "knn_k33", "adj_sparse_random", "dense_n97"]


def _spec(name):
    return N97 if name == "dense_n97" else cases.SPECS[name]


def blocks(n):
    """An uneven partition of the rows whose inner boundaries are no multiple of 16 or 32."""
    if n >= 97:
        return [(0, 33), (33, 70), (70, n)]
    if n >= 70:
        return [(0, 33), (33, n)]
    a, b = n // 3 + 1, (2 * n) // 3 + 1
    return [(0, a), (a, b), (b, n)]


def zero_outside(g, rows):
    out = np.zeros_like(g)
    out[:, rows[0]:rows[1]] = g[:, rows[0]:rows[1]]
    return out


# ----------------------------------------------------------------------------- C ABI (CPU)


def _desc(nat, **kw):
    base = dict(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=2, N=1024, C=3, dim=32, edge_dim=0, label_dim=0,
                num_labels=0, m_dim=16, fourier=0, k=0, flags=nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS,
                valid_radius=1e30, clamp=0.0, row_begin=0, row_end=0, reserved=0)
    base.update(kw)
    return nat.LayerDesc(**base)


def _bwd_bytes(nat, **kw):
    nb = C.c_size_t()
    rc = nat.load().egnn_layer_backward_workspace_bytes(C.byref(_desc(nat, **kw)), C.byref(nb))
    return rc, nb.value


def test_flag_opts_row_blocks_into_the_backward(nat):
    part = nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS | nat.FLAG_ROW_PARTIAL_GRADS
    for k in (0, 20):
        for rows in ((0, 256), (33, 70), (700, 1024), (5, 5)):
            assert _bwd_bytes(nat, k=k, row_begin=rows[0], row_end=rows[1], flags=part)[0] == 0, (k, rows)
            assert _bwd_bytes(nat, k=k, row_begin=rows[0], row_end=rows[1])[0] == -3, (k, rows)      # no flag: as before
        # what the backward cannot run stays rejected with the flag
        assert _bwd_bytes(nat, k=k, row_begin=33, row_end=70, flags=part, dtype=nat.DTYPE_BF16)[0] == -3
        assert _bwd_bytes(nat, k=k, row_begin=33, row_end=70, flags=part, label_dim=4, num_labels=17)[0] == -3
        assert _bwd_bytes(nat, k=k, row_begin=33, row_end=70, flags=part, dtype=nat.DTYPE_F64, m_dim=32)[0] == -3
        # the flag over all rows sizes exactly what the unflagged call does
        assert _bwd_bytes(nat, k=k, flags=part) == _bwd_bytes(nat, k=k)
        assert _bwd_bytes(nat, k=k, row_end=1024, flags=part) == _bwd_bytes(nat, k=k)


@pytest.mark.parametrize("dtype,es,m_dim,fourier,edge_dim", [("DTYPE_F32", 4, 16, 0, 0), ("DTYPE_F64", 8, 16, 0, 0),
                                                             ("DTYPE_F32", 4, 32, 2, 3), ("DTYPE_F64", 8, 24, 2, 3)])
def test_per_pair_workspace_scales_with_the_block(nat, dtype, es, m_dim, fourier, edge_dim):
    """Dense N = 1024, a block of R = 256 rows: the backward workspace shrinks by exactly the per-pair record and pre2 of
    the other N - R rows (each region rounded up to 256 bytes), i.e. per-pair memory per rank goes as R / N."""
    B, N, R = 2, 1024, 256
    kw = dict(dtype=getattr(nat, dtype), m_dim=m_dim, fourier=fourier, edge_dim=edge_dim)
    part = nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS | nat.FLAG_ROW_PARTIAL_GRADS
    rc_full, full = _bwd_bytes(nat, **kw)
    rc_blk, blk = _bwd_bytes(nat, row_begin=300, row_end=300 + R, flags=part, **kw)
    assert rc_full == 0 and rc_blk == 0
    mp_ = 16 if m_dim <= 16 else 32
    q = 2 * fourier + 1 + edge_dim
    rec = int(math.ceil((mp_ + 2 * q + 2) / 4) * 4)                  # record width per pair
    up = lambda x: (x + 255) // 256 * 256
    per_pair = lambda rows: up(B * rows * N * rec * es) + up(B * rows * N * mp_ * es)
    assert full - blk == per_pair(N) - per_pair(R)


# ----------------------------------------------------------------------------- one layer on the GPU


def _module_grads(case, dtype, gf, gx, rows=None, mod=None, neighbors=None, slot_edges=None, seed=None):
    """Forward + backward of the module with `_rows=rows` and loss sum(fo * gf) + sum(xo * gx) -> flat gradients."""
    mod = mod if mod is not None else util.make_module(case, dtype)
    mod.requires_grad_(True)
    mod.zero_grad(set_to_none=True)
    ins = case["inputs"]
    t = lambda name: util.to_torch(ins.get(name), dtype, "cuda")
    feats, coors = t("feats").requires_grad_(True), t("coors").requires_grad_(True)
    leaves = {"in.feats": feats, "in.coors": coors}
    kw = dict(mask=t("mask"), _rows=rows)
    edges = None
    if slot_edges is not None:
        kw["neighbor_edges"] = leaves["in.neighbor_edges"] = util.to_torch(slot_edges, dtype, "cuda").requires_grad_(True)
    elif ins.get("edges") is not None:
        edges = leaves["in.edges"] = t("edges").requires_grad_(True)
    if neighbors is not None:
        kw["neighbors"] = torch.from_numpy(neighbors).cuda()
    elif ins.get("adj_mat") is not None:
        kw["adj_mat"] = t("adj_mat")
    g_f, g_x = (torch.from_numpy(np.asarray(g)).to(device="cuda", dtype=dtype) for g in (gf, gx))
    if seed is not None:
        torch.manual_seed(seed)
    with torch.enable_grad():
        fo, xo = mod(feats, coors, edges, **kw)
        ((fo * g_f).sum() + (xo * g_x).sum()).backward()
    out = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    for k, p in mod.named_parameters():
        out[f"p.{k}"] = (torch.zeros_like(p) if p.grad is None else p.grad).double().cpu().numpy()
    return out


@functools.lru_cache(maxsize=None)
def _case(name):
    return cases.build_case(_spec(name))


@functools.lru_cache(maxsize=None)
def _oracle(name, rows):
    """Oracle gradient of block `rows` (None = all rows): the cotangents zeroed outside it."""
    case = _case(name)
    gf, gx = cases.upstream_grads(case)
    if rows is not None:
        gf, gx = zero_outside(gf, rows), zero_outside(gx, rows)
    ins = case["inputs"]
    return cases.flatten_grads(G.egnn_layer_backward(case["params"], case["cfg"], ins["feats"], ins["coors"], ins.get("edges"),
                                                     ins.get("mask"), ins.get("adj_mat"), gf, gx))


def _sum(dicts):
    return {k: sum(d[k] for d in dicts) for k in dicts[0]}


_BLOCK_PARAMS = [(n, dt, mode) for n in BLOCK_CASES for dt in (torch.float64, torch.float32) for mode in ("saved", "recompute")
                 if not (n == "dense_mdim32" and dt == torch.float64)]     # fp64 m_dim 32: over the backward's shared memory


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype,mode", _BLOCK_PARAMS,
                         ids=[f"{n}-{str(d)[6:]}-{m}" for n, d, m in _BLOCK_PARAMS])
def test_block_gradients_match_the_oracle_and_sum_to_the_full_gradient(name, dtype, mode, monkeypatch):
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    case = _case(name)
    tol = util.grad_tol(case, dtype)
    gf, gx = cases.upstream_grads(case)
    mod = util.make_module(case, dtype)
    parts = []
    for rows in blocks(case["spec"]["N"]):
        got = _module_grads(case, dtype, zero_outside(gf, rows), zero_outside(gx, rows), rows=rows, mod=mod)
        util.compare(got, _oracle(name, rows), tol, f"{name} block {rows} vs oracle")
        parts.append(got)
    total = _sum(parts)
    util.compare(total, _oracle(name, None), tol, f"{name} sum of blocks vs oracle")
    util.compare(total, _module_grads(case, dtype, gf, gx, mod=mod), tol, f"{name} sum of blocks vs whole-layer backward")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_everything", "knn_edges_mask", "dense_n97"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_flag_over_all_rows_matches_the_unflagged_backward(name, dtype):
    case = _case(name)
    gf, gx = cases.upstream_grads(case)
    mod = util.make_module(case, dtype)
    n = case["spec"]["N"]
    util.compare(_module_grads(case, dtype, gf, gx, rows=(0, n), mod=mod), _module_grads(case, dtype, gf, gx, mod=mod),
                 util.grad_tol(case, dtype), f"{name} (0, N) with the flag vs without")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_everything", "knn_edges_mask"])
@pytest.mark.parametrize("rows", [(5, 5), (0, 0)], ids=["5-5", "0-0"])
def test_empty_block_gives_zero_gradients(name, rows):
    """Nothing of the layer is evaluated: the parameters get 0, the inputs only the identity of the untouched rows."""
    case = _case(name)
    gf, gx = cases.upstream_grads(case)
    got = _module_grads(case, torch.float64, gf, gx, rows=rows)
    assert np.array_equal(got["in.feats"], gf) and np.array_equal(got["in.coors"], gx)
    for k, v in got.items():
        if k not in ("in.feats", "in.coors"):
            assert not v.any(), k
    got = _module_grads(case, torch.float64, zero_outside(gf, rows), zero_outside(gx, rows), rows=rows)
    assert all(not v.any() for v in got.values())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16], ids=["fp64", "fp32", "bf16"])
@pytest.mark.parametrize("rows", [(5, 5), (0, 0)], ids=["5-5", "0-0"])
def test_empty_block_forward_is_the_identity_with_and_without_grad(rows, dtype):
    """An empty range returns the inputs unchanged, whatever the grad mode."""
    case = _case("dense_xavier" if dtype == torch.bfloat16 else "dense_everything")
    mod = util.make_module(case, dtype)
    ins = case["inputs"]
    f, x = util.to_torch(ins["feats"], dtype, "cuda"), util.to_torch(ins["coors"], dtype, "cuda")
    e = util.to_torch(ins.get("edges"), dtype, "cuda")
    m = util.to_torch(ins.get("mask"), dtype, "cuda")
    with torch.no_grad():
        fo, xo = mod(f, x, e, mask=m, _rows=rows)
    assert torch.equal(fo, f) and torch.equal(xo, x)
    if dtype != torch.bfloat16:
        with torch.enable_grad():
            fg, xg = mod(f.clone().requires_grad_(True), x.clone().requires_grad_(True), e, mask=m, _rows=rows)
        assert torch.equal(fg.detach(), f) and torch.equal(xg.detach(), x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_everything", "knn_edges_mask", "dense_no_feats", "dense_no_coors"])
def test_rows_call_differentiates_as_block_plus_identity(name):
    """A loss over ALL rows of a `_rows` call (the rows outside the block are the inputs, returned unchanged): the
    gradient is the block's oracle gradient plus the identity outside the block."""
    case = _case(name)
    gf, gx = cases.upstream_grads(case)
    rows = blocks(case["spec"]["N"])[1]
    want = dict(_oracle(name, rows))
    for key, g in (("in.feats", gf), ("in.coors", gx)):
        want[key] = want[key] + g - zero_outside(g, rows)
    got = _module_grads(case, torch.float64, gf, gx, rows=rows)
    util.compare(got, want, util.grad_tol(case, torch.float64), f"{name} _rows={rows} with identity rows")


def _caller_lists(B, N, k, e, seed=5):
    rs = np.random.RandomState(seed)
    nb = np.stack([np.stack([rs.permutation(N)[:k] for _ in range(N)]) for _ in range(B)]).astype(np.int64)
    nb[:, ::3, -2:] = -1                           # every third node has two empty slots
    nb[0, 5, :] = -1                               # one node has no neighbour at all
    return nb, rs.randn(B, N, k, e)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,mode", [(torch.float64, "saved"), (torch.float64, "recompute"), (torch.float32, "saved"),
                                        (torch.float32, "recompute")],
                         ids=["fp64-saved", "fp64-recompute", "fp32-saved", "fp32-recompute"])
def test_caller_lists_with_per_slot_edges_sum_to_the_full_backward(dtype, mode, monkeypatch):
    """Edge-list mode with `neighbor_edges` (no oracle takes per-slot edges): the blocks sum to the whole-layer backward,
    which tests/test_slot_edges.py pins to its per-slot reference."""
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    spec = dict(kind="layer", cfg=dict(dim=16, edge_dim=3, soft_edges=True, m_pool_method="mean"), B=2, N=37, seed=71,
                init="xavier", mask="padded")
    case = cases.build_case(spec)
    nb, se = _caller_lists(2, 37, 9, 3)
    gf, gx = cases.upstream_grads(case)
    mod = util.make_module(case, dtype)
    parts = [_module_grads(case, dtype, zero_outside(gf, r), zero_outside(gx, r), rows=r, mod=mod, neighbors=nb, slot_edges=se)
             for r in blocks(37)]
    full = _module_grads(case, dtype, gf, gx, mod=mod, neighbors=nb, slot_edges=se)
    util.compare(_sum(parts), full, util.grad_tol(case, dtype), "per-slot edges: sum of blocks vs whole layer")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_everything", "knn_edges_mask"])
def test_dropout_blocks_with_one_seed_sum_to_the_full_gradient(name):
    """Dropout masks are keyed on global indices: blocks drawn with the seed of the whole-graph call sum to its gradient."""
    case = _case(name)
    gf, gx = cases.upstream_grads(case)
    mod = util.make_module(case, torch.float64, dropout=0.2).train()
    parts = [_module_grads(case, torch.float64, zero_outside(gf, r), zero_outside(gx, r), rows=r, mod=mod, seed=11)
             for r in blocks(case["spec"]["N"])]
    full = _module_grads(case, torch.float64, gf, gx, mod=mod, seed=11)
    other = _module_grads(case, torch.float64, gf, gx, mod=mod, seed=12)
    assert max(np.abs(other[k] - full[k]).max() for k in full) > 1e-3          # the masks matter
    util.compare(_sum(parts), full, util.grad_tol(case, torch.float64), f"{name} dropout: sum of blocks vs whole layer")


# ----------------------------------------------------------------------------- row sharding over ranks (gloo, CPU)


class _OracleLayer(torch.autograd.Function):
    """The numpy oracle as a differentiable row block: rows r0:r1 are the layer's output, the other rows its input."""

    @staticmethod
    def forward(ctx, feats, coors, rows, cfg, keys, edges, mask, *params):
        P = {k: p.detach().numpy() for k, p in zip(keys, params)}
        f_np, x_np = feats.detach().numpy(), coors.detach().numpy()
        e_np = None if edges is None else edges.numpy()
        m_np = None if mask is None else mask.numpy()
        f, x = O.egnn_layer_forward(P, cfg, f_np, x_np, edges=e_np, mask=m_np, rows=rows)
        F, X = f_np.copy(), x_np.copy()
        F[:, rows[0]:rows[1]] = f
        X[:, rows[0]:rows[1]] = x
        ctx.args = (P, cfg, f_np, x_np, e_np, m_np, rows, keys, [p.shape for p in params])
        return torch.from_numpy(F), torch.from_numpy(X)

    @staticmethod
    def backward(ctx, g_f, g_x):
        P, cfg, f_np, x_np, e_np, m_np, rows, keys, shapes = ctx.args
        g_f, g_x = g_f.numpy(), g_x.numpy()
        r = G.egnn_layer_backward(P, cfg, f_np, x_np, e_np, m_np, None, zero_outside(g_f, rows), zero_outside(g_x, rows))
        g_feats = r["feats"] + g_f - zero_outside(g_f, rows)
        g_coors = r["coors"] + g_x - zero_outside(g_x, rows)
        grads = [torch.from_numpy(np.asarray(r["params"][k]).reshape(s)) for k, s in zip(keys, shapes)]
        return (torch.from_numpy(g_feats), torch.from_numpy(g_coors), None, None, None, None, None, *grads)


def _oracle_chain_grads(case, layers, gf, gx):
    """Full-graph oracle gradient of layers applied in sequence -> (d feats, d coors, [param grads per layer])."""
    ins, cfg = case["inputs"], case["cfg"]
    e, m = ins.get("edges"), ins.get("mask")
    acts = [(ins["feats"], ins["coors"])]
    for P in layers[:-1]:
        acts.append(O.egnn_layer_forward(P, cfg, *acts[-1], edges=e, mask=m))
    pgrads = [None] * len(layers)
    for li in reversed(range(len(layers))):
        r = G.egnn_layer_backward(layers[li], cfg, *acts[li], e, m, None, gf, gx)
        gf, gx, pgrads[li] = r["feats"], r["coors"], r["params"]
    return gf, gx, pgrads


def _gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from egnn_pytorch_b200 import parallel
        for name in ("knn_edges_mask", "dense_mask_padded"):
            case = cases.build_case(cases.SPECS[name])
            cfg, ins = case["cfg"], case["inputs"]
            layers = [case["params"], cases.gen_layer_params(cfg, np.random.RandomState(99), "xavier")]
            gf, gx = cases.upstream_grads(case)
            want_f, want_x, want_p = _oracle_chain_grads(case, layers, gf, gx)
            n = ins["feats"].shape[1]
            r0, r1 = parallel.shard_range(n, rank, world)
            keys = sorted(layers[0])
            params = [[torch.nn.Parameter(torch.from_numpy(np.asarray(P[k], np.float64))) for k in keys] for P in layers]
            edges = None if ins.get("edges") is None else torch.from_numpy(ins["edges"])
            mask = None if ins.get("mask") is None else torch.from_numpy(ins["mask"])
            f = torch.from_numpy(ins["feats"][:, r0:r1].copy()).requires_grad_(True)
            x = torch.from_numpy(ins["coors"][:, r0:r1].copy()).requires_grad_(True)
            h, c = f, x
            for ps in params:
                fn = lambda fa, xa, rows, ps=ps: _OracleLayer.apply(fa, xa, rows, cfg, keys, edges, mask, *ps)
                h, c = parallel.row_sharded_layer_call(fn, h, c, n)
            loss = (h * torch.from_numpy(gf[:, r0:r1])).sum() + (c * torch.from_numpy(gx[:, r0:r1])).sum()
            loss.backward()
            flat = [p for ps in params for p in ps]
            parallel.allreduce_gradients(flat, bucket_bytes=4096)
            # relative to max(1, |want|): the second (xavier) layer drives some gradients to ~1e5
            rel = lambda got, want: np.abs(got - want).max() / max(1.0, np.abs(want).max())
            assert rel(f.grad.numpy(), want_f[:, r0:r1]) <= 1e-11, name
            assert rel(x.grad.numpy(), want_x[:, r0:r1]) <= 1e-11, name
            for li, ps in enumerate(params):
                for k, p in zip(keys, ps):
                    err = rel(p.grad.numpy(), np.asarray(want_p[li][k]).reshape(p.shape))
                    assert err <= 1e-11, (name, li, k, err)
        q.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _spawn(worker, port_base, timeout):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = port_base + os.getpid() % 2000
    procs = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=timeout) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] == "ok" for r in res), res


def test_row_sharded_training_world2_gloo():
    """Two chained layers over two ranks, the compute an oracle-backed autograd Function: after backward and
    allreduce_gradients, the local input gradients and the parameter gradients equal the full-graph oracle gradient."""
    _spawn(_gloo_worker, 31500, 300)


# ----------------------------------------------------------------------------- row sharding over two GPUs


def _single_gpu_grads(mods, feats, coors, gf, gx, kw):
    f, x = feats.clone().requires_grad_(True), coors.clone().requires_grad_(True)
    h, c = f, x
    with torch.enable_grad():
        for m in mods:
            h, c = m(h, c, **kw)
        ((h * gf).sum() + (c * gx).sum()).backward()
    return f.grad, x.grad, [[p.grad.clone() for p in m.parameters()] for m in mods]


def _close(got, want, what):
    scale = max(1.0, float(want.abs().max()))
    err = float((got.double() - want.double()).abs().max()) / scale
    assert math.isfinite(err) and err <= 5e-4, (what, err)


def _nccl_worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        from egnn_pytorch_b200 import parallel
        for name in ("dense_mask_padded", "knn_edges_mask"):
            case = cases.build_case(cases.SPECS[name])
            ins = {k: util.to_torch(v, torch.float32, dev) for k, v in case["inputs"].items()}
            b, n, d = ins["feats"].shape
            r0, r1 = parallel.shard_range(n, rank, world)
            gf, gx = (torch.from_numpy(g).to(dev, torch.float32) for g in cases.upstream_grads(case))
            kw = dict(mask=ins.get("mask"), edges=ins.get("edges"))
            for how, depth in (("peer", 3), ("call", 2)):
                mods = [util.make_module(case, torch.float32, device=dev).requires_grad_(True) for _ in range(depth)]
                refs = [util.make_module(case, torch.float32, device=dev).requires_grad_(True) for _ in range(depth)]
                want_f, want_x, want_p = _single_gpu_grads(refs, ins["feats"], ins["coors"], gf, gx, kw)
                f = ins["feats"][:, r0:r1].clone().requires_grad_(True)
                x = ins["coors"][:, r0:r1].clone().requires_grad_(True)
                h, c = f, x
                with torch.enable_grad():
                    if how == "peer":
                        _, payload = parallel.row_payload_layout(n, x.shape[-1], d, 4, b)
                        comm = parallel.PeerComm(payload)
                        for m in mods:                   # depth 3: the double-buffered gather wraps before backward
                            h, c = parallel.row_sharded_layer_peer(comm, m, h, c, n, **kw)
                    else:
                        for m in mods:
                            h, c = parallel.row_sharded_layer_call(
                                lambda fa, xa, rows, m=m: m(fa, xa, kw["edges"], mask=kw["mask"], _rows=rows), h, c, n)
                    ((h * gf[:, r0:r1]).sum() + (c * gx[:, r0:r1]).sum()).backward()
                parallel.allreduce_gradients([p for m in mods for p in m.parameters()])
                torch.cuda.synchronize(dev)
                if how == "peer":
                    assert comm.status() == 0
                    comm.close()
                _close(f.grad, want_f[:, r0:r1], f"{name} {how} feats")
                _close(x.grad, want_x[:, r0:r1], f"{name} {how} coors")
                for li, m in enumerate(mods):
                    for p, w in zip(m.parameters(), want_p[li]):
                        _close(p.grad, w, f"{name} {how} layer {li} parameter")
        dist.barrier()
        q.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_row_sharded_training_two_gpus():
    """Three layers through the peer-memory gather (its double buffer wraps under grad) and two through the
    torch.distributed gather, dense and kNN in fp32: after backward and allreduce_gradients the local input gradients
    and the parameter gradients equal single-GPU training of the whole graph."""
    _spawn(_nccl_worker, 31700, 900)

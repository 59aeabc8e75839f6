"""Parity of the CUDA path (through the module API -> C ABI -> sm_90a kernels) against the
oracle and the committed reference outputs.  Needs an H100: `pytest -m gpu`.

Tolerances (stated per SURVEY.md section 8(c)):
  fp64 kernels : atol 1e-9,  rtol 1e-9   (same algebra, different summation order)
  fp32 kernels : atol 2e-5,  rtol 1e-4   vs the fp64 oracle (the reference's own fp32-vs-fp64
                 deviation is <= 5e-6 at these sizes, BASELINE.md section 2)
"""
import glob
import os

import numpy as np
import pytest
import torch

import cases
import util

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = list(cases.SPECS)
TOL = {torch.float64: dict(atol=1e-9, rtol=1e-9), torch.float32: dict(atol=2e-5, rtol=1e-4)}


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", NAMES)
def test_cuda_matches_oracle_and_golden(name, dtype):
    case = cases.build_case(cases.SPECS[name])
    mod = util.make_module(case, dtype)
    kw = dict(return_coor_changes=True) if case["kind"] == "network" else {}
    out = util.run_module(mod, case, dtype, **kw)
    want = cases.run_oracle(case)
    util.assert_close(out[0], want[0], what=f"{name} feats vs oracle", **TOL[dtype])
    util.assert_close(out[1], want[1], what=f"{name} coors vs oracle", **TOL[dtype])
    g = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    if not bool(g["tie_dependent"]):
        util.assert_close(out[0], g["feats"], what=f"{name} feats vs reference", **TOL[dtype])
        util.assert_close(out[1], g["coors"], what=f"{name} coors vs reference", **TOL[dtype])
        if case["kind"] == "network":
            util.assert_close(torch.stack(out[2]), g["coor_changes"], what=f"{name} coor_changes", **TOL[dtype])
    layer = mod.layers[0][1] if case["kind"] == "network" else mod
    assert layer.last_path == ("fp64-simt" if dtype == torch.float64 else "fp32-simt")


def test_cpu_tensors_are_staged_and_returned_on_cpu():
    """The reference's tests call the layer with CPU float64 tensors (tests/test_equivariance.py:28)."""
    case = cases.build_case(cases.SPECS["dense_edges"])
    mod = util.make_module(case, torch.float64, device="cpu")
    out = util.run_module(mod, case, torch.float64, device="cpu")
    assert out[0].device.type == "cpu" and out[0].dtype == torch.float64
    want = cases.run_oracle(case)
    util.assert_close(out[0], want[0], atol=1e-9, rtol=1e-9)
    util.assert_close(out[1], want[1], atol=1e-9, rtol=1e-9)


def test_inputs_not_mutated_and_param_update_is_seen():
    case = cases.build_case(cases.SPECS["dense_basic"])
    mod = util.make_module(case, torch.float32)
    ins = case["inputs"]
    f = util.to_torch(ins["feats"], torch.float32, "cuda")
    x = util.to_torch(ins["coors"], torch.float32, "cuda")
    f0, x0 = f.clone(), x.clone()
    o1 = mod(f, x)
    assert torch.equal(f, f0) and torch.equal(x, x0)
    with torch.no_grad():
        mod.edge_mlp[3].bias.add_(0.25)      # in-place update must invalidate the packed cache
    o2 = mod(f, x)
    assert not torch.allclose(o1[0], o2[0])
    case["params"]["edge_mlp.3.bias"] = case["params"]["edge_mlp.3.bias"] + 0.25
    want = cases.run_oracle(case)
    util.assert_close(o2[0], want[0], atol=2e-5, rtol=1e-4)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("k,n,masked,adj", [(1, 5, False, False), (8, 300, True, False), (32, 1000, False, False),
                                            (7, 64, True, True), (40, 333, True, False), (64, 64, False, False)])
def test_knn_select_kernel(k, n, masked, adj, dtype):
    """egnn_knn_select alone vs the oracle's ranking + stable smallest-k (egnn_pytorch.py:237-260)."""
    import ctypes as C
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    rs = np.random.RandomState(k * 1000 + n)
    B, Cd = 2, 3
    # coordinates on a 1/8 grid: squared distances are exact in fp32 and fp64, so the ranking is
    # independent of FMA contraction, and ties (incl. coincident nodes) are frequent -> this pins
    # the lowest-index tie rule
    coors = np.round(rs.standard_normal((B, n, Cd)) * 8) / 8
    mask = (rs.uniform(size=(B, n)) < 0.85) if masked else None
    adjm = cases.chain_adjacency(n, True) if adj else None
    cfg = cases.O.layer_cfg(dim=4, num_nearest_neighbors=k, valid_radius=1.0)
    idx, ok, _ = cases.O.neighbour_selection(cfg, coors.astype(np.float32 if dtype == torch.float32 else np.float64),
                                             mask, adjm)
    tc = torch.from_numpy(coors).to("cuda", dtype).contiguous()
    tm = None if mask is None else torch.from_numpy(mask).to("cuda", torch.uint8).contiguous()
    ta = None if adjm is None else torch.from_numpy(adjm).to("cuda", torch.uint8).contiguous()
    oi = torch.empty((B, n, k), dtype=torch.int32, device="cuda")
    oo = torch.empty((B, n, k), dtype=torch.uint8, device="cuda")
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    rc = lib.egnn_knn_select(nat.DTYPE_F64 if dtype == torch.float64 else nat.DTYPE_F32, B, n, Cd, k, p(tc), p(tm), p(ta),
                             0, 1.0, p(oi), p(oo), None)
    assert rc == 0, nat.strerror(rc)
    torch.cuda.synchronize()
    got = oi.cpu().numpy()
    np.testing.assert_array_equal(got, idx)
    np.testing.assert_array_equal(oo.cpu().numpy().astype(bool), ok)


@pytest.mark.parametrize("n,deg,batched", [(40, 3, False), (70, 2, True), (33, 4, False), (257, 3, False)])
def test_adj_expand_kernel(n, deg, batched):
    import ctypes as C
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    rs = np.random.RandomState(n)
    B = 2
    if batched:
        a = rs.uniform(size=(B, n, n)) < 0.04
        a = a | a.transpose(0, 2, 1)
    else:
        a = cases.chain_adjacency(n, n % 2 == 0)
    want_adj, want_lab = cases.O.adjacency_degrees(a, deg, B)
    ta = torch.from_numpy(a).to("cuda", torch.uint8).contiguous()
    adj_out = torch.empty((B, n, n), dtype=torch.uint8, device="cuda")
    lab = torch.empty((B, n, n), dtype=torch.uint8, device="cuda")
    mx = torch.zeros(1, dtype=torch.int32, device="cuda")
    nb = C.c_size_t()
    assert lib.egnn_adj_workspace_bytes(B, n, C.byref(nb)) == 0
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = lib.egnn_adj_expand(B, n, deg, p(ta), 1 if batched else 0, p(adj_out), p(lab), p(mx), p(ws), nb.value, None)
    assert rc == 0, nat.strerror(rc)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(adj_out.cpu().numpy().astype(bool), want_adj)
    np.testing.assert_array_equal(lab.cpu().numpy().astype(np.int64), want_lab)
    assert int(mx.item()) == int(want_adj.sum(-1).max())


def test_host_buffer_entry_matches_device_entry():
    """egnn_layer_forward_host (the e2e entry bench.py times) == the device-pointer entry."""
    import ctypes as C
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    case = cases.build_case(cases.SPECS["dense_mask_padded"])
    mod = util.make_module(case, torch.float32)
    out = util.run_module(mod, case, torch.float32)
    ins = case["inputs"]
    st = mod._staged(torch.device("cuda", 0), torch.float32)
    T = st["tensors"]
    packed = next(iter(st["packed"].values()))
    B, N, d = ins["feats"].shape
    desc = nat.LayerDesc(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=B, N=N, C=3, dim=d, edge_dim=mod.edge_dim, label_dim=0,
                         num_labels=0, m_dim=16, fourier=0, k=0, flags=mod._flags(), valid_radius=3e38, clamp=0.0,
                         row_begin=0, row_end=0, reserved=0)
    w = nat.LayerWeights(**{f: (T[f].data_ptr() if f in T else None) for f in nat.WEIGHT_FIELDS})
    hf = torch.from_numpy(ins["feats"]).float().pin_memory()
    hx = torch.from_numpy(ins["coors"]).float().pin_memory()
    he = torch.from_numpy(ins["edges"]).float().pin_memory()
    hm = torch.from_numpy(ins["mask"]).to(torch.uint8).pin_memory()
    of, ox = torch.empty_like(hf).pin_memory(), torch.empty_like(hx).pin_memory()
    io = nat.LayerIO(feats=hf.data_ptr(), coors=hx.data_ptr(), edges=he.data_ptr(), edge_labels=None,
                     mask=hm.data_ptr(), adj=None, feats_out=of.data_ptr(), coors_out=ox.data_ptr())
    rc = lib.egnn_layer_forward_host(C.byref(desc), C.byref(w), C.c_void_p(packed.data_ptr()), C.byref(io), None)
    assert rc == 0, nat.strerror(rc)
    assert torch.equal(of, out[0].cpu()) and torch.equal(ox, out[1].cpu())


def test_error_behaviour():
    from egnn_pytorch_b200 import EGNN
    layer = EGNN(dim=8, num_nearest_neighbors=9).cuda()
    with pytest.raises(RuntimeError):           # k > N: torch.topk raises in the reference too
        layer(torch.randn(1, 5, 8, device="cuda"), torch.randn(1, 5, 3, device="cuda"))
    with pytest.raises(AssertionError):
        EGNN(dim=8, m_pool_method="max")
    with pytest.raises(AssertionError):
        EGNN(dim=8, update_feats=False, update_coors=False)
    layer = EGNN(dim=8, edge_dim=2).cuda()
    with pytest.raises(AssertionError):
        layer(torch.randn(1, 5, 8, device="cuda"), torch.randn(1, 5, 3, device="cuda"))   # edges missing


@pytest.mark.parametrize("name", ["dense_mask_padded", "net_c3_small", "net_c5_small"])
def test_cuda_graph_capture_replays_the_forward(name):
    """egnn_pytorch_b200.GraphedForward: the whole forward is stream-ordered and sync-free, hence capturable."""
    from egnn_pytorch_b200 import GraphedForward
    case = cases.build_case(cases.SPECS[name])
    mod = util.make_module(case, torch.float32)
    ins = {k: util.to_torch(v, torch.float32, "cuda") for k, v in case["inputs"].items()}
    if case["kind"] == "network":
        args = (ins["feats"], ins["coors"])
        kw = {k: ins[k] for k in ("adj_mat", "edges", "mask") if k in ins}
    else:
        args = (ins["feats"], ins["coors"]) + ((ins["edges"],) if "edges" in ins else ())
        kw = {k: ins[k] for k in ("mask", "adj_mat") if k in ins}
    eager = mod(*args, **kw)
    fast = GraphedForward(mod, *args, **kw)
    out = fast(*args)
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
    # new coordinates through the same graph
    x2 = args[1] * 1.25 + 0.5
    args2 = (args[0], x2) + tuple(args[2:])
    out2 = [t.clone() for t in fast(*args2)]
    eager2 = mod(*args2, **kw)
    assert torch.equal(out2[0], eager2[0]) and torch.equal(out2[1], eager2[1])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_edge_list_mode_matches_the_select_path(dtype):
    """`neighbors=`: (1) the lists egnn_knn_select would pick reproduce the kNN forward bit for bit; (2) a chain given
    as an edge_index (with -1 padding at the ends) equals `only_sparse_neighbors` on the chain adjacency."""
    import ctypes as C
    from egnn_pytorch_b200 import EGNN, edge_index_to_neighbors, _native as nat
    lib = nat.load()
    torch.manual_seed(0)
    B, N, d, k = 2, 60, 64, 6
    feats = torch.randn(B, N, d, device="cuda").to(dtype)
    coors = torch.randn(B, N, 3, device="cuda")
    mask = torch.ones(B, N, dtype=torch.bool, device="cuda")
    layer = EGNN(dim=d, num_nearest_neighbors=k).to(dtype).cuda().eval()
    f0, x0 = layer(feats, coors, mask=mask)
    idx = torch.empty(B, N, k, dtype=torch.int32, device="cuda")
    rc = lib.egnn_knn_select(nat.DTYPE_F32, B, N, 3, k, C.c_void_p(coors.data_ptr()), None, None, 0, float("inf"),
                             C.c_void_p(idx.data_ptr()), None, None)
    assert rc == 0
    f1, x1 = layer(feats, coors, mask=mask, neighbors=idx)
    assert torch.equal(f0, f1) and torch.equal(x0, x1)
    # chain graph as an edge list
    i = torch.arange(N, device="cuda")
    src = torch.cat([i, i[:-1], i[1:]]); dst = torch.cat([i, i[1:], i[:-1]])        # self, i-1 -> i, i+1 -> i
    nbrs = edge_index_to_neighbors(torch.stack([src, dst]), N).expand(B, -1, -1)
    assert nbrs.shape[-1] == 3 and int((nbrs < 0).sum()) == 2 * B
    sparse = EGNN(dim=d, only_sparse_neighbors=True).to(dtype).cuda().eval()
    sparse.load_state_dict(layer.state_dict())
    adj = (i[:, None] - i[None, :]).abs() <= 1
    f2, x2 = sparse(feats, coors, mask=mask, adj_mat=adj)
    f3, x3 = layer(feats, coors, mask=mask, neighbors=nbrs)
    tol = 2e-2 if dtype == torch.bfloat16 else 1e-5          # same edges, different slot order -> different summation order
    assert float((f2.float() - f3.float()).abs().max()) <= tol * float(f2.float().abs().max())
    assert float((x2 - x3).abs().max()) <= tol

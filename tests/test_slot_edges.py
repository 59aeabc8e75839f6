"""Edge-list mode with edge features per neighbour slot: `EGNN.forward(..., neighbors=, neighbor_edges=)`
(EGNN_FLAG_EDGES_PER_SLOT), where slot s of node i carries the features of the edge neighbors[b, i, s] -> i and no
[B, N, N, edge_dim] tensor exists.

The per-slot oracle below restates the flat per-edge form of `oracle.egnn_oracle.egnn_layer_forward_edge_list` (one
row per existing slot, scatter-add onto the receiving node) in float64 torch on the CPU, with the edge input taken
from the slot instead of the pair; its gradients are autograd's.  It is pinned to the numpy edge-list oracles
(forward and gradient) on duplicate-free lists, and to central finite differences on lists where one node lists the
same neighbour twice with different features -- the case no dense tensor can express.

CPU: the oracle, `edge_index_to_neighbors(..., edge_attr=)`, descriptor validation through ctypes, misuse errors.
GPU: forward (fp64 / fp32 / bf16) and backward (fp64 / fp32, W2 silu(pre1) saved or recomputed) against the oracle,
bit-equality with the dense-edge call on gathered features, dropout, a 131,072-node graph, row ranges and the
host-buffer entry."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import cases
import util
from oracle import egnn_oracle as O
from oracle import egnn_oracle_grad as G
from util import nat  # noqa: F401  (module-scoped fixture)

CASES = {
    # name: (layer cfg, B, N, k, C, mask?).  Comments: the bf16 list kernel mode and the bwd2 channel instantiation
    # (Q = 2F + 1 + edge_dim per-pair channels: QR = 8 for Q <= 8, QR = 0 above).
    "edges3_mask":     (dict(dim=16, edge_dim=3), 2, 24, 6, 3, True),                        # TK_EDGES, Q 4
    "edges4_soft_mean": (dict(dim=32, edge_dim=4, soft_edges=True, m_pool_method="mean"), 2, 30, 9, 3, True),  # TK_EDGES
    "fourier_gen":     (dict(dim=16, edge_dim=2, fourier_features=2, norm_feats=True), 1, 28, 7, 3, False),  # TK_GEN, Q 7
    "edges9_normc":    (dict(dim=8, edge_dim=9, norm_coors=True), 2, 26, 5, 3, True),        # TK_GEN (edge_dim > 4), Q 10
    "c2_clamp":        (dict(dim=16, edge_dim=2, coor_weights_clamp_value=0.5), 2, 20, 4, 2, False),  # TK_GEN (C = 2)
    "c5_mean":         (dict(dim=8, edge_dim=3, m_pool_method="mean"), 1, 22, 6, 5, True),  # TK_GEN (C = 5)
    "k40":             (dict(dim=8, edge_dim=2, soft_edges=True), 1, 60, 40, 3, True),     # two SIMT slot passes
    "k33_mdim24":      (dict(dim=12, m_dim=24, edge_dim=1), 2, 37, 33, 3, False),          # fp64: 32-wide accumulators
}


def build(name, seed=0, dups=True):
    """-> (case, neighbour lists [B,N,k] int64, per-slot edge features [B,N,k,e]).  Lists hold no self edges; every
    third node has two empty (-1) slots, node 5 of graph 0 has none at all, and with `dups` node 4 lists its first
    neighbour twice (with different features).  Empty slots carry random features, which must be ignored."""
    cfg, B, N, k, Cd, with_mask = CASES[name]
    spec = dict(kind="layer", cfg=cfg, B=B, N=N, C=Cd, seed=2000 + seed, init="xavier", mask="padded" if with_mask else None)
    case = cases.build_case(spec)
    rs = np.random.RandomState(300 + seed)
    nb = np.stack([np.stack([rs.permutation(np.delete(np.arange(N), i))[:k] for i in range(N)]) for _ in range(B)])
    nb = nb.astype(np.int64)
    nb[:, ::3, -2:] = -1
    nb[0, 5, :] = -1
    if dups:
        nb[:, 4, 1] = nb[:, 4, 0]
    se = rs.randn(B, N, k, cfg["edge_dim"])
    return case, nb, se


def gathered(edges, nb):
    """Per-slot features read from a dense [B,N,N,e] tensor: slot s of row i = edges[b, i, nb[b,i,s]] (0 if empty)."""
    B, N, k = nb.shape
    se = np.asarray(edges)[np.arange(B)[:, None, None], np.arange(N)[None, :, None], np.maximum(nb, 0)]
    return np.where((nb >= 0)[..., None], se, 0.0)


# ----------------------------------------------------------------------------- the per-slot oracle


def _t(x):
    return x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.float64))


def slot_oracle(params, cfg, feats, coors, neighbors, slot_edges, mask=None):
    """The layer on caller lists with per-slot edge features, float64, flat per-edge form: exactly
    `egnn_oracle.egnn_layer_forward_edge_list` with `slot_edges[eb, ei, es]` in place of `edges[eb, ei, ej]`.
    Inputs may be torch tensors that require grad."""
    P = {k: _t(v) for k, v in params.items()}
    feats, coors, slot_edges = _t(feats), _t(coors), _t(slot_edges)
    nb = torch.as_tensor(np.asarray(neighbors)).long()
    b, n, d = feats.shape
    k = nb.shape[-1]
    eb, ei, es = torch.nonzero(nb >= 0, as_tuple=True)            # one row per existing slot
    ej = nb[eb, ei, es]
    rel = coors[eb, ei] - coors[eb, ej]
    dist = (rel ** 2).sum(-1)
    F = cfg["fourier_features"]
    if F > 0:
        sc = dist[:, None] / (2.0 ** torch.arange(F, dtype=torch.float64))
        dfeat = torch.cat([torch.sin(sc), torch.cos(sc), dist[:, None]], -1)
    else:
        dfeat = dist[:, None]
    edge_in = torch.cat([feats[eb, ei], feats[eb, ej], dfeat, slot_edges[eb, ei, es]], -1)
    lin = lambda x, key: x @ P[key + ".weight"].T + P[key + ".bias"]
    m = TF.silu(lin(TF.silu(lin(edge_in, "edge_mlp.0")), "edge_mlp.3"))
    if cfg["soft_edges"]:
        m = m * torch.sigmoid(lin(m, "edge_gate.0"))
    live = None
    if mask is not None:
        mk = torch.as_tensor(np.asarray(mask)).bool()
        live = mk[eb, ei] & mk[eb, ej]
    coors_out = coors
    if cfg["update_coors"]:
        w = lin(TF.silu(lin(m, "coors_mlp.0")), "coors_mlp.3")[:, 0]
        if live is not None:
            w = torch.where(live, w, torch.zeros_like(w))
        cv = cfg["coor_weights_clamp_value"]
        if cv is not None:
            w = w.clamp(-cv, cv)
        rel_n = rel
        if cfg["norm_coors"]:
            rel_n = rel / torch.linalg.vector_norm(rel, dim=-1, keepdim=True).clamp_min(1e-8) * P["coors_norm.scale"]
        coors_out = coors.index_put((eb, ei), w[:, None] * rel_n, accumulate=True)
    feats_out = feats
    if cfg["update_feats"]:
        mm = m if live is None else torch.where(live[:, None], m, torch.zeros_like(m))
        m_i = feats.new_zeros((b, n, m.shape[-1])).index_put((eb, ei), mm, accumulate=True)
        if cfg["m_pool_method"] == "mean":
            if live is not None:
                cnt = feats.new_zeros((b, n, 1)).index_put((eb, ei), live[:, None].double(), accumulate=True)
                m_i = torch.where(cnt == 0, torch.zeros_like(m_i), m_i / cnt.clamp_min(1e-8))
            else:
                m_i = m_i / k
        normed = TF.layer_norm(feats, (d,), P["node_norm.weight"], P["node_norm.bias"], 1e-5) if cfg["norm_feats"] else feats
        h1 = TF.silu(lin(torch.cat([normed, m_i], -1), "node_mlp.0"))
        feats_out = lin(h1, "node_mlp.3") + feats
    return feats_out, coors_out


def slot_oracle_grads(case, nb, se, gf=None, gx=None):
    """Gradients of sum(feats_out * gf) + sum(coors_out * gx) through the per-slot oracle, flat like util.module_grads:
    'in.feats', 'in.coors', 'in.neighbor_edges', 'p.<state-dict key>'."""
    ins = case["inputs"]
    if gf is None:
        gf, gx = cases.upstream_grads(case)
    leaves = {"in.feats": _t(ins["feats"]).requires_grad_(True), "in.coors": _t(ins["coors"]).requires_grad_(True),
              "in.neighbor_edges": _t(se).clone().requires_grad_(True)}
    P = {k: _t(v).clone().requires_grad_(True) for k, v in case["params"].items()}
    with torch.enable_grad():
        fo, xo = slot_oracle(P, case["cfg"], leaves["in.feats"], leaves["in.coors"], nb, leaves["in.neighbor_edges"],
                             ins.get("mask"))
        ((fo * _t(gf)).sum() + (xo * _t(gx)).sum()).backward()
    out = {k: v.grad.numpy() for k, v in leaves.items()}
    out.update({f"p.{k}": v.grad.numpy() for k, v in P.items()})
    return out


# ----------------------------------------------------------------------------- CPU: the oracle


@pytest.mark.parametrize("name", sorted(CASES))
def test_slot_oracle_equals_the_dense_edge_list_oracle(name):
    case, nb, _ = build(name, dups=False)
    ins = case["inputs"]
    want = O.egnn_layer_forward_edge_list(case["params"], case["cfg"], ins["feats"], ins["coors"], nb, ins["edges"], ins.get("mask"))
    got = slot_oracle(case["params"], case["cfg"], ins["feats"], ins["coors"], nb, gathered(ins["edges"], nb), ins.get("mask"))
    assert np.abs(got[0].numpy() - want[0]).max() <= 1e-12 and np.abs(got[1].numpy() - want[1]).max() <= 1e-12


@pytest.mark.parametrize("name", ["edges3_mask", "edges4_soft_mean", "fourier_gen", "edges9_normc", "c5_mean"])
def test_slot_oracle_gradient_equals_the_dense_edge_list_gradient_oracle(name):
    """Duplicate-free lists: every gradient equals the numpy backward oracle, and the slot gradients scattered onto
    [B,N,N,e] equal its dense d/d edges."""
    case, nb, _ = build(name, dups=False)
    ins = case["inputs"]
    gf, gx = cases.upstream_grads(case)
    got = slot_oracle_grads(case, nb, gathered(ins["edges"], nb), gf, gx)
    g = G.egnn_layer_backward(case["params"], case["cfg"], ins["feats"], ins["coors"], ins["edges"], ins.get("mask"), None,
                              gf, gx, neighbors=nb)
    B, N, k = nb.shape
    dense = np.zeros_like(ins["edges"])
    bi, ii, si = np.nonzero(nb >= 0)
    np.add.at(dense, (bi, ii, nb[bi, ii, si]), got["in.neighbor_edges"][bi, ii, si])
    want = {"in.feats": g["feats"], "in.coors": g["coors"], "dense_edges": g["edges"]}
    want.update({f"p.{k}": v for k, v in g["params"].items()})
    got = dict(got, dense_edges=dense)
    assert not np.abs(got.pop("in.neighbor_edges")[nb < 0]).any()             # empty slots get no gradient
    util.compare(got, want, 1e-10, f"{name}: per-slot oracle gradient vs numpy gradient oracle")


@pytest.mark.parametrize("name", ["edges3_mask", "edges4_soft_mean", "fourier_gen", "c2_clamp", "c5_mean"])
def test_slot_oracle_gradient_matches_finite_differences_with_a_duplicate_neighbour(name):
    case, nb, se = build(name)
    assert (nb[:, 4, 0] == nb[:, 4, 1]).all() and not np.allclose(se[:, 4, 0], se[:, 4, 1])
    ins, cfg, P = case["inputs"], case["cfg"], case["params"]
    rs = np.random.RandomState(11)
    gf, gx = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape)
    g = slot_oracle_grads(case, nb, se, gf, gx)

    def loss(feats, coors, e, params):
        fo, xo = slot_oracle(params, cfg, feats, coors, nb, e, ins.get("mask"))
        return float((fo.numpy() * gf).sum() + (xo.numpy() * gx).sum())

    vf, vx, ve = rs.randn(*ins["feats"].shape), rs.randn(*ins["coors"].shape), rs.randn(*se.shape)
    vp = {k: rs.randn(*np.shape(v)) for k, v in P.items()}
    eps = 1e-6
    shift = lambda s: loss(ins["feats"] + s * eps * vf, ins["coors"] + s * eps * vx, se + s * eps * ve,
                           {k: np.asarray(v) + s * eps * vp[k] for k, v in P.items()})
    fd = (shift(1) - shift(-1)) / (2 * eps)
    an = ((g["in.feats"] * vf).sum() + (g["in.coors"] * vx).sum() + (g["in.neighbor_edges"] * ve).sum()
          + sum((g[f"p.{k}"] * vp[k]).sum() for k in P))
    assert abs(fd - an) <= 2e-6 * max(1.0, abs(an)), (fd, an)
    # the two slots of the duplicate carry their own gradients (where the pair is not masked out)
    gd = g["in.neighbor_edges"][:, 4]
    assert not any(np.allclose(gd[b, 0], gd[b, 1]) for b in range(len(gd)) if np.abs(gd[b, :2]).any())


# ----------------------------------------------------------------------------- CPU: edge_index_to_neighbors, ABI, misuse


def test_edge_index_to_neighbors_places_edge_attr_in_its_slot():
    from egnn_pytorch_b200 import edge_index_to_neighbors
    # node 0 <- 1, 2, 3 (in that order after a stable sort), node 2 <- 0, node 3 <- 0, 1; node 1 has none
    src = torch.tensor([1, 0, 2, 0, 3, 1])
    dst = torch.tensor([0, 2, 0, 3, 0, 3])
    ei = torch.stack([src, dst])
    attr = torch.arange(12, dtype=torch.float64).reshape(6, 2).requires_grad_(True)
    torch.set_grad_enabled(True)            # (this test differentiates; the suite's default is inference mode)
    nb_plain = edge_index_to_neighbors(ei, 4)
    nb, ne = edge_index_to_neighbors(ei, 4, edge_attr=attr)
    assert torch.equal(nb, nb_plain) and nb.dtype == torch.int32
    assert nb.tolist() == [[[1, 2, 3], [-1, -1, -1], [0, -1, -1], [0, 1, -1]]]
    assert ne.shape == (1, 4, 3, 2)
    for e in range(6):                                  # each attribute sits in its edge's slot
        i, j = int(dst[e]), int(src[e])
        s = nb[0, i].tolist().index(j)
        assert torch.equal(ne[0, i, s], attr[e])
    assert not ne[0][nb[0] < 0].any()                   # empty slots are zero
    # truncation at k = 2: node 0 keeps its first two edges (1, 2), node 3 both
    nb2, ne2 = edge_index_to_neighbors(ei, 4, k=2, edge_attr=attr)
    assert torch.equal(nb2, edge_index_to_neighbors(ei, 4, k=2)) and nb2.tolist() == [[[1, 2], [-1, -1], [0, -1], [0, 1]]]
    assert torch.equal(ne2, ne[:, :, :2])
    # gradients flow back to edge_attr, truncated edges get none
    (ne2 * torch.arange(1, 17, dtype=torch.float64).reshape(1, 4, 2, 2)).sum().backward()
    g = attr.grad
    assert torch.equal(g[4], torch.zeros(2, dtype=torch.float64))          # edge 3 -> 0 was truncated
    assert torch.equal(g[0], torch.tensor([1.0, 2.0], dtype=torch.float64))  # edge 1 -> 0: node 0 slot 0
    assert torch.equal(g[5], torch.tensor([15.0, 16.0], dtype=torch.float64))  # edge 1 -> 3: node 3 slot 1


def test_descriptor_validation_of_the_per_slot_flag(nat):
    """Through ctypes, without a device: the flag needs k > 0 and edge_dim > 0, and caller lists at the call."""
    lib = nat.load()
    nb = C.c_size_t()
    uf_uc = nat.FLAG_UPDATE_FEATS | nat.FLAG_UPDATE_COORS
    good = dict(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=2, N=16, C=3, dim=32, edge_dim=4, label_dim=0,
                num_labels=0, m_dim=16, fourier=0, k=8, flags=uf_uc | nat.FLAG_EDGES_PER_SLOT, valid_radius=1e30,
                clamp=0.0, row_begin=0, row_end=0, reserved=0)
    assert nat.ABI_VERSION == lib.egnn_abi_version() == 4
    rc = lambda fn, **kw: getattr(lib, fn)(C.byref(nat.LayerDesc(**dict(good, **kw))), C.byref(nb))
    for fn in ("egnn_layer_packed_bytes", "egnn_layer_workspace_bytes", "egnn_layer_backward_workspace_bytes"):
        assert rc(fn) == 0, fn
        assert rc(fn, k=0) == -2, fn
        assert rc(fn, edge_dim=0) == -2, fn
        assert rc(fn, flags=uf_uc, k=0) == 0 and rc(fn, flags=uf_uc, edge_dim=0) == 0, fn
    assert rc("egnn_layer_packed_bytes", dtype=nat.DTYPE_BF16) == 0
    # the calls reject a descriptor with the flag and no caller lists before touching any pointer (dummy, aligned)
    p = 1 << 12
    d = nat.LayerDesc(**good)
    w = nat.LayerWeights(**{f: p for f in nat.WEIGHT_FIELDS})
    io = nat.LayerIO(feats=p, coors=p, edges=p, feats_out=p, coors_out=p, nbr_idx=None)
    assert lib.egnn_layer_forward(C.byref(d), C.byref(w), C.c_void_p(p), C.byref(io), C.c_void_p(p), 1 << 20, None) == -2
    grads = nat.LayerGrads(g_feats_out=p, g_coors_out=p, g_feats=p, g_coors=p, g_edges=p,
                           w=nat.LayerWeightGrads(**{f: p for f in nat.WEIGHT_FIELDS}))
    assert lib.egnn_layer_backward(C.byref(d), C.byref(w), C.c_void_p(p), C.byref(io), C.c_void_p(p), C.byref(grads),
                                   C.c_void_p(p), 1 << 20, None) == -2


def test_misuse_of_neighbor_edges_raises_before_any_launch(monkeypatch):
    from egnn_pytorch_b200 import EGNN, _native

    def no_launch():
        raise AssertionError("the library was reached")

    monkeypatch.setattr(_native, "load", no_launch)
    mod = EGNN(dim=8, edge_dim=3)
    B, N, k = 2, 10, 4
    f, x = torch.randn(B, N, 8), torch.randn(B, N, 3)
    nbl = torch.randint(0, N, (B, N, k))
    ne = torch.randn(B, N, k, 3)
    with pytest.raises(ValueError, match="needs neighbors"):
        mod(f, x, neighbor_edges=ne)
    with pytest.raises(ValueError, match="not both"):
        mod(f, x, torch.randn(B, N, N, 3), neighbors=nbl, neighbor_edges=ne)
    for bad in (torch.randn(B, N, k + 1, 3), torch.randn(B, N, k, 2), torch.randn(B, N - 1, k, 3)):
        with pytest.raises(ValueError, match=r"\(B, N, k, edge_dim\)"):
            mod(f, x, neighbors=nbl, neighbor_edges=bad)
    with pytest.raises(ValueError, match="edge_dim > 0"):
        EGNN(dim=8)(f, x, neighbors=nbl, neighbor_edges=torch.randn(B, N, k, 0))


# ----------------------------------------------------------------------------- GPU


def _inputs(case, nb, se, dtype, device="cuda"):
    ins = case["inputs"]
    t = lambda v: util.to_torch(v, dtype, device)
    return t(ins["feats"]), t(ins["coors"]), t(ins.get("mask")), torch.from_numpy(nb).to(device), t(se)


def _run(case, nb, se, dtype):
    mod = util.make_module(case, dtype)
    f, x, m, n, e = _inputs(case, nb, se, dtype)
    with torch.no_grad():
        out = mod(f, x, mask=m, neighbors=n, neighbor_edges=e)
    return mod, out


def _bf16_case(case, se):
    rnd = lambda v: torch.from_numpy(np.asarray(v, np.float64)).bfloat16().double().numpy()
    case["params"] = {k: rnd(v) for k, v in case["params"].items()}
    for key in ("feats", "coors", "edges"):
        case["inputs"][key] = rnd(case["inputs"][key])
    return case, rnd(se)


def _tc_covers(case, k):
    cfg = case["cfg"]
    return cfg["dim"] % 8 == 0 and k <= 32 and cfg["m_dim"] == 16


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_forward_matches_slot_oracle(name, dtype):
    case, nb, se = build(name)
    ins = case["inputs"]
    want = slot_oracle(case["params"], case["cfg"], ins["feats"], ins["coors"], nb, se, ins.get("mask"))
    _, got = _run(case, nb, se, dtype)
    tol = util.TOL[dtype]
    util.assert_close(got[0], want[0].numpy(), what=f"{name} feats", **tol)
    util.assert_close(got[1], want[1].numpy(), what=f"{name} coors", **tol)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_bf16_matches_slot_oracle(name):
    case, nb, se = build(name)
    case, se = _bf16_case(case, se)
    ins = case["inputs"]
    want = [w.numpy() for w in slot_oracle(case["params"], case["cfg"], ins["feats"], ins["coors"], nb, se, ins.get("mask"))]
    mod, got = _run(case, nb, se, torch.bfloat16)
    ferr = util.max_err(got[0], want[0]) / max(1.0, float(np.abs(want[0]).max()))
    cerr = util.max_err(got[1], want[1]) / max(1.0, float(np.abs(want[1] - ins["coors"]).max()))
    if _tc_covers(case, nb.shape[-1]):
        assert mod.last_path == "bf16-tc"
    assert ferr < 1e-2 and cerr < 1e-2, (name, mod.last_path, ferr, cerr)


GATHER_CASES = ["edges3_mask", "edges4_soft_mean", "fourier_gen", "edges9_normc", "c5_mean", "k40"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GATHER_CASES)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16], ids=["fp64", "fp32", "bf16"])
def test_gathered_features_give_the_dense_edge_outputs_bit_for_bit(name, dtype):
    case, nb, _ = build(name, dups=False)
    edges = case["inputs"]["edges"]
    mod = util.make_module(case, dtype)
    f, x, m, n, e = _inputs(case, nb, gathered(edges, nb), dtype)
    with torch.no_grad():
        dense = mod(f, x, util.to_torch(edges, dtype, "cuda"), mask=m, neighbors=n)
        path = mod.last_path
        slot = mod(f, x, mask=m, neighbors=n, neighbor_edges=e)
    assert mod.last_path == path
    assert torch.equal(dense[0], slot[0]) and torch.equal(dense[1], slot[1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", GATHER_CASES)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_gathered_features_backward_equals_the_dense_edge_backward(name, dtype):
    """The slot gradients scattered onto [B,N,N,e] equal the dense call's d/d edges exactly: the dense call adds each
    entry once onto zero, and both read the same per-pair record.  That record is bit-reproducible for these shapes --
    at most two bwd2 channel CTAs add into it (Hp <= 256; two addends onto zero commute) and the node-MLP backward that
    feeds bwd1 runs one K split (2 dim <= 64) -- which the asserts below pin.  Every other gradient is summed with
    atomics in an arbitrary order (g_coors in bwd3, dL/dB_j in bwd2 at ~k atomics per (j, h), the per-CTA weight
    gradients), in both calls independently, so they are compared at the fp32 gradient tolerance of the suite
    (util.grad_tol: 5e-4 of max(1, |max|)) and at 1e-11 in fp64."""
    case, nb, _ = build(name, dups=False)
    edges = case["inputs"]["edges"]
    cfg = case["cfg"]
    Hp = -(-2 * (2 * cfg["dim"] + 2 * cfg["fourier_features"] + 1 + cfg["edge_dim"]) // 8) * 8
    assert Hp <= 256 and 2 * cfg["dim"] <= 64, (Hp, cfg["dim"])

    def grads(slot):
        mod = util.make_module(case, dtype).requires_grad_(True)
        f, x, m, n, e = _inputs(case, nb, gathered(edges, nb) if slot else edges, dtype)
        f.requires_grad_(True); x.requires_grad_(True); e.requires_grad_(True)
        gf, gx = (torch.from_numpy(g).to(device="cuda", dtype=dtype) for g in cases.upstream_grads(case))
        with torch.enable_grad():
            fo, xo = mod(f, x, mask=m, neighbors=n, neighbor_edges=e) if slot else mod(f, x, e, mask=m, neighbors=n)
            ((fo * gf).sum() + (xo * gx).sum()).backward()
        out = {"in.feats": f.grad, "in.coors": x.grad, "edges": e.grad}
        out.update({f"p.{k}": p.grad for k, p in mod.named_parameters()})
        return out

    dense, slot = grads(False), grads(True)
    ge = slot.pop("edges")
    assert ge.shape == nb.shape + (edges.shape[-1],) and not ge[torch.from_numpy(nb < 0).cuda()].any()
    scattered = torch.zeros_like(dense["edges"])
    bi, ii, si = (torch.from_numpy(a).cuda() for a in np.nonzero(nb >= 0))
    scattered[bi, ii, torch.from_numpy(nb).cuda()[bi, ii, si]] = ge[bi, ii, si]
    assert torch.equal(scattered, dense.pop("edges"))
    tol = 1e-11 if dtype == torch.float64 else util.grad_tol(case, dtype)
    util.compare({k: v.double().cpu().numpy() for k, v in slot.items()},
                 {k: v.double().cpu().numpy() for k, v in dense.items()}, tol, f"{name} slot vs dense gradients")


@functools.lru_cache(maxsize=None)
def _oracle_grads(name):
    case, nb, se = build(name)
    return case, nb, se, slot_oracle_grads(case, nb, se)


def module_slot_grads(case, nb, se, dtype):
    mod = util.make_module(case, dtype).requires_grad_(True)
    f, x, m, n, e = _inputs(case, nb, se, dtype)
    leaves = {"in.feats": f.requires_grad_(True), "in.coors": x.requires_grad_(True), "in.neighbor_edges": e.requires_grad_(True)}
    gf, gx = (torch.from_numpy(g).to(device="cuda", dtype=dtype) for g in cases.upstream_grads(case))
    with torch.enable_grad():
        fo, xo = mod(f, x, mask=m, neighbors=n, neighbor_edges=e)
        ((fo * gf).sum() + (xo * gx).sum()).backward()
    out = {k: v.grad.double().cpu().numpy() for k, v in leaves.items()}
    out.update({f"p.{k}": p.grad.double().cpu().numpy() for k, p in mod.named_parameters()})
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("dtype,mode", [(torch.float64, "saved"), (torch.float64, "recompute"), (torch.float32, "saved"),
                                        (torch.float32, "recompute")],
                         ids=["fp64-saved", "fp64-recompute", "fp32-saved", "fp32-recompute"])
def test_backward_matches_slot_oracle(name, dtype, mode, monkeypatch):
    if mode == "recompute":
        monkeypatch.setenv("EGNN_B200_SAVE_PAIR_MB", "0")
    case, nb, se, want = _oracle_grads(name)
    got = module_slot_grads(case, nb, se, dtype)
    assert not got["in.neighbor_edges"][nb < 0].any()
    util.compare(got, want, util.grad_tol(case, dtype), f"{name} {mode} vs per-slot oracle")


@pytest.mark.gpu
def test_dropout_gradient_with_neighbor_edges_matches_finite_differences():
    """Training-mode dropout (masks keyed on the pair (b*N + i)*N + j, so the duplicate's two slots share one): with a
    fixed seed the fp64 analytic gradient, d/d neighbor_edges included, equals central finite differences."""
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(3)
    cfg = dict(dim=12, dropout=0.25, edge_dim=3, soft_edges=True, m_pool_method="mean")
    mod = EGNN(**cfg).double().cuda().train()
    for p in mod.parameters():
        if p.dim() == 2:
            torch.nn.init.xavier_normal_(p)
    B, N, k = 2, 14, 5
    case_nb = np.stack([np.stack([np.random.RandomState(40 + i).permutation(np.delete(np.arange(N), i))[:k]
                                  for i in range(N)]) for _ in range(B)])
    case_nb[:, ::3, -1] = -1
    case_nb[:, 4, 1] = case_nb[:, 4, 0]
    nbl = torch.from_numpy(case_nb).cuda()
    torch.manual_seed(4)
    f = torch.randn(B, N, 12, device="cuda", dtype=torch.float64)
    x = torch.randn(B, N, 3, device="cuda", dtype=torch.float64)
    e = torch.randn(B, N, k, 3, device="cuda", dtype=torch.float64)
    mask = torch.ones(B, N, dtype=torch.bool, device="cuda"); mask[-1, -2:] = False
    gf, gx = torch.randn_like(f), torch.randn_like(x)

    def loss(ff, xx, ee):
        torch.manual_seed(99)
        fo, xo = mod(ff, xx, mask=mask, neighbors=nbl, neighbor_edges=ee)
        return (fo * gf).sum() + (xo * gx).sum()

    fr, xr, er = (t.clone().requires_grad_(True) for t in (f, x, e))
    with torch.enable_grad():
        loss(fr, xr, er).backward()
    params = list(mod.parameters())
    vf, vx, ve = torch.randn_like(f), torch.randn_like(x), torch.randn_like(e)
    vp = [torch.randn_like(p) for p in params]
    an = float((fr.grad * vf).sum() + (xr.grad * vx).sum() + (er.grad * ve).sum() + sum((p.grad * v).sum() for p, v in zip(params, vp)))
    eps = 1e-6

    def shifted(sign):
        with torch.no_grad():
            for p, v in zip(params, vp):
                p.add_(sign * eps * v)
            mod.invalidate_cache()
            val = float(loss(f + sign * eps * vf, x + sign * eps * vx, e + sign * eps * ve))
            for p, v in zip(params, vp):
                p.sub_(sign * eps * v)
            mod.invalidate_cache()
        return val

    fd = (shifted(+1) - shifted(-1)) / (2 * eps)
    assert np.isfinite(an) and abs(fd - an) <= 2e-4 * max(1.0, abs(an)), (fd, an)
    assert float(er.grad[nbl < 0].abs().max()) == 0.0


@pytest.mark.gpu
def test_large_sparse_graph_equals_the_same_graph_as_a_batch():
    """B = 1, N = 131,072 nodes in 2,048 disjoint blocks of 64, k = 16 in-block neighbours (with -1 slots), edge_dim = 4:
    one graph, and the same graph as a batch [2048, 64] with re-indexed lists.  Any 32-bit overflow of i*N or i*k
    addressing shows up as a difference.  Peak memory must stay below 4 GiB: any O(N^2) buffer needs at least
    N^2 = 17.2 GB (one byte per pair); a dense fp32 edge tensor would need 275 GB."""
    from egnn_pytorch_b200 import EGNN
    torch.manual_seed(0)
    nblk, blk, k, e_dim, dim = 2048, 64, 16, 4, 32
    N = nblk * blk
    g = torch.Generator(device="cpu").manual_seed(1)
    local = torch.argsort(torch.rand(nblk, blk, blk, generator=g), dim=-1)[..., :k]     # in-block neighbours
    local[:, ::5, -3:] = -1
    local[:, 7, :] = -1                                                                 # nodes with no neighbours
    glob = torch.where(local >= 0, local + (torch.arange(nblk) * blk)[:, None, None], local).reshape(1, N, k)
    feats = torch.randn(1, N, dim, device="cuda")
    coors = torch.randn(1, N, 3, device="cuda")
    ne = torch.randn(1, N, k, e_dim, device="cuda")
    mod = EGNN(dim=dim, edge_dim=e_dim).cuda()
    for p in mod.parameters():
        if p.dim() == 2:
            torch.nn.init.xavier_normal_(p)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()

    def train_run(as_batch):
        shape = (nblk, blk) if as_batch else (1, N)
        f = feats.reshape(*shape, dim).clone().requires_grad_(True)
        x = coors.reshape(*shape, 3).clone().requires_grad_(True)
        e = ne.reshape(*shape, k, e_dim).clone().requires_grad_(True)
        lists = (local if as_batch else glob).cuda()
        mod.zero_grad(set_to_none=True)
        with torch.enable_grad():
            fo, xo = mod(f, x, neighbors=lists, neighbor_edges=e)
            (fo.square().mean() + xo.square().mean()).backward()
        out = {"feats": fo.reshape(1, N, dim), "coors": xo.reshape(1, N, 3), "g.feats": f.grad.reshape(1, N, dim),
               "g.coors": x.grad.reshape(1, N, 3), "g.edges": e.grad.reshape(1, N, k, e_dim)}
        out.update({f"g.{n}": p.grad for n, p in mod.named_parameters()})
        return {n: v.detach() for n, v in out.items()}

    one, batch = train_run(False), train_run(True)
    assert mod.last_path == "fp32-simt"
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 4 * 2 ** 30, f"peak {peak / 2 ** 30:.2f} GiB"
    for n in one:
        scale = max(1.0, float(batch[n].abs().max()))
        err = float((one[n] - batch[n]).abs().max()) / scale
        # forward: same arithmetic per row; gradients: atomics in another order (the suite's fp32 gradient tolerance)
        assert err <= (1e-6 if n in ("feats", "coors") else util.grad_tol(None, torch.float32)), (n, err)
    # bf16 forward
    mod_bf = mod.to(torch.bfloat16)
    with torch.no_grad():
        a = mod_bf(feats.bfloat16(), coors, neighbors=glob.cuda(), neighbor_edges=ne.bfloat16())
        assert mod_bf.last_path == "bf16-tc"
        bt = mod_bf(feats.bfloat16().reshape(nblk, blk, dim), coors.reshape(nblk, blk, 3), neighbors=local.cuda(),
                    neighbor_edges=ne.bfloat16().reshape(nblk, blk, k, e_dim))
    for u, v in zip(a, bt):
        u, v = u.float(), v.float().reshape(u.shape)
        assert float((u - v).abs().max()) <= 1e-2 * max(1.0, float(u.abs().max()))
    assert torch.cuda.max_memory_allocated() - base < 4 * 2 ** 30


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_row_range_is_bit_identical_to_the_full_forward(dtype):
    case, nb, se = build("edges4_soft_mean")
    if dtype == torch.bfloat16:
        case, se = _bf16_case(case, se)
    mod = util.make_module(case, dtype)
    f, x, m, n, e = _inputs(case, nb, se, dtype)
    N = nb.shape[1]
    with torch.no_grad():
        full = mod(f, x, mask=m, neighbors=n, neighbor_edges=e)
        path = mod.last_path
        for r0, r1 in [(0, 11), (11, 23), (23, N)]:
            fr, xr = mod(f, x, mask=m, neighbors=n, neighbor_edges=e, _rows=(r0, r1))
            assert mod.last_path == path
            assert torch.equal(fr[:, r0:r1], full[0][:, r0:r1]) and torch.equal(xr[:, r0:r1], full[1][:, r0:r1])
    if dtype == torch.bfloat16:
        assert path == "bf16-tc"


@pytest.mark.gpu
def test_host_buffer_entry_with_per_slot_edges_matches_device_entry():
    from egnn_pytorch_b200 import _native as nat
    lib = nat.load()
    case, nb, se = build("edges3_mask")
    mod = util.make_module(case, torch.float32)
    f, x, m, n, e = _inputs(case, nb, se, torch.float32)
    with torch.no_grad():
        out = mod(f, x, mask=m, neighbors=n, neighbor_edges=e)
    st = mod._staged(torch.device("cuda", torch.cuda.current_device()), torch.float32)
    T = st["tensors"]
    packed = next(iter(st["packed"].values()))
    B, N, k = nb.shape
    desc = nat.LayerDesc(abi_version=nat.ABI_VERSION, dtype=nat.DTYPE_F32, B=B, N=N, C=3, dim=mod.dim, edge_dim=mod.edge_dim,
                         label_dim=0, num_labels=0, m_dim=16, fourier=0, k=k, flags=mod._flags() | nat.FLAG_EDGES_PER_SLOT,
                         valid_radius=float("inf"), clamp=0.0, row_begin=0, row_end=0, reserved=0)
    w = nat.LayerWeights(**{fl: (T[fl].data_ptr() if fl in T else None) for fl in nat.WEIGHT_FIELDS})
    hf, hx, he = (t.cpu().contiguous().pin_memory() for t in (f, x, e))
    hm = m.to(torch.uint8).cpu().pin_memory()
    hn = n.to(torch.int32).cpu().pin_memory()
    of, ox = torch.empty_like(hf).pin_memory(), torch.empty_like(hx).pin_memory()
    io = nat.LayerIO(feats=hf.data_ptr(), coors=hx.data_ptr(), edges=he.data_ptr(), edge_labels=None, mask=hm.data_ptr(),
                     adj=None, feats_out=of.data_ptr(), coors_out=ox.data_ptr(), nbr_idx=hn.data_ptr())
    torch.cuda.synchronize()
    rc = lib.egnn_layer_forward_host(C.byref(desc), C.byref(w), C.c_void_p(packed.data_ptr()), C.byref(io), None)
    assert rc == 0, nat.strerror(rc)
    assert torch.equal(of, out[0].cpu()) and torch.equal(ox, out[1].cpu())

"""Neighbour lists longer than 32 slots on the bf16 tensor-core path, against the rounding-matched reference.

tc_knn_kernel runs a row's k > 32 slots in groups of 32 in the same warp (its WIDE instantiations, DESIGN.md section
5).  The case table mirrors the launch choice in `geometry` and test_table_covers_every_boundary holds it to:
  k = 33 / 63 / 64 / 65 / 96 / 127 / 128 / 200 (2 - 7 groups, partial and full last groups); the lean, edges and
  generic instantiations at 8 and 16 rows per CTA; partial last CTAs; no lattice, a box and a cell.
Caller lists carry -1 slots at random, on the last slot of a group, as a whole group in the middle of a row, and as a
whole row; some rows hold their own node.  Options: mean pooling with and without a mask, clamp, soft edges,
CoorsNorm, per-slot edges (edges and generic), fourier features, C = 2 and C = 5.  Lists from the layer's own select
(num_nearest_neighbors = 64 with valid_radius and a mask; plain, under a box and under a tilted cell) and from
EGNN_Network's only_sparse_neighbors over an expanded adjacency (degree labels) run on the tensor cores without a
warning.  Row ranges, per-slot edges against the dense tensor, and a diagonal cell against its box are bit for bit.

The gates and their tolerances are test_gpu_tc_boundaries.py's (`TOL`), plus its gate against the fp64 oracle."""
import contextlib
import warnings

import numpy as np
import pytest
import torch

import cases
import launch_geometry as LG
import tc_reference as T
import test_gpu_tc_boundaries as TB
import torch_reference as R
import util
from oracle import egnn_oracle as O

L, NW = "layer", "network"
TOL = TB.TOL
BOX3 = TB.BOX3

CASES = {
    # lean: 2 groups (the second holds 1 slot) at 8 rows; 3 full groups at 16 rows
    "w33_lean8":        dict(kind=L, cfg=dict(dim=32), B=2, N=203, k=33, seed=801, holes=True),
    "w96_lean16_clamp": dict(kind=L, cfg=dict(dim=344, coor_weights_clamp_value=3.0), B=1, N=150, k=96, seed=802,
                             holes=True),
    # edges: per-slot edges, 2 groups (the second one slot short); dense edges, 4 groups (the last one short) at 16 rows
    "w63_edges8_slot":  dict(kind=L, cfg=dict(dim=64, edge_dim=4), B=2, N=150, k=63, seed=803, holes=True,
                             slot_edges=True, mask="padded"),
    "w127_edges16":     dict(kind=L, cfg=dict(dim=280, edge_dim=4, soft_edges=True), B=1, N=150, k=127, seed=804,
                             holes=True, mask="random"),
    # generic: fourier + mean without a mask; C = 5 with edges, soft edges and CoorsNorm; a row range at 16 rows with
    # per-slot edges and mean over a mask; C = 2 over 7 groups
    "w64_gen8_mean":    dict(kind=L, cfg=dict(dim=32, fourier_features=2, m_pool_method="mean"), B=2, N=100, k=64,
                             seed=805, holes=True),
    "w65_gen8_c5":      dict(kind=L, cfg=dict(dim=32, edge_dim=2, soft_edges=True, norm_coors=True), B=2, N=77, C=5,
                             k=65, seed=806, mask="random", holes=True),
    "w128_gen16_rows":  dict(kind=L, cfg=dict(dim=264, fourier_features=2, edge_dim=1, m_pool_method="mean"), B=2,
                             N=150, k=128, seed=807, holes=True, slot_edges=True, mask="padded", rows=(19, 140)),
    "w200_gen8_c2":     dict(kind=L, cfg=dict(dim=32, coor_weights_clamp_value=1.0, m_pool_method="mean"), B=2, N=230,
                             C=2, k=200, seed=808, holes=True, mask="padded"),
    # c4's layer (dim 256, edge_dim 4) on lists of 96 with per-slot edges
    "w96_c4":           dict(kind=L, cfg=dict(dim=256, edge_dim=4), B=2, N=4096, k=96, seed=809, slot_edges=True,
                             holes=True, check=[(0, 16), (2040, 2056), (4080, 4096)]),
}
# the same boundaries under a box ("wb_") and a cell ("wc_")
for _n in ("w33_lean8", "w63_edges8_slot", "w96_lean16_clamp", "w127_edges16", "w64_gen8_mean", "w128_gen16_rows"):
    _s = CASES[_n]
    _box, _cell = (BOX3, "tilt") if _s["B"] == 1 else ("per_graph", "per_graph")
    CASES[f"wb_{_n[1:]}"] = dict(_s, box=_box, seed=_s["seed"] + 100)
    CASES[f"wc_{_n[1:]}"] = dict(_s, cell=_cell, seed=_s["seed"] + 200)
CASES["wc_c2_gen8"] = dict(kind=L, cfg=dict(dim=32, m_pool_method="mean"), B=2, N=120, C=2, k=40, seed=830,
                           holes=True, cell="c2", mask="padded")


def geometry(spec, sms=LG.H100_SMS):
    """What the launch code runs a case with: tc_knn_kernel<MODE, ROWS, PBC, WIDE = k > 32>, ceil(k / 32) groups."""
    g = LG.tc_layer(spec["kind"], spec["cfg"], spec["B"], spec["N"], C=spec.get("C", 3), k=spec["k"],
                    rows=spec.get("rows"), sms=sms)
    return dict(g, lattice=TB.lattice_kind(spec))


def test_table_covers_every_boundary():
    geo = {n: geometry(s) for n, s in CASES.items()}
    assert all(g["supported"] and g["wide"] for g in geo.values())
    assert {g["k"] for g in geo.values()} >= {33, 63, 64, 65, 96, 127, 128, 200}
    assert {g["groups"] for g in geo.values()} >= {2, 3, 4, 7}
    assert {g["last_group"] for g in geo.values()} >= {1, 31, 32}
    for lat in (None, "box", "cell"):
        sub = {n: g for n, g in geo.items() if g["lattice"] == lat}
        assert {g["kernel"] for g in sub.values()} >= {
            f"tc_knn<{m},{r}>" for m in ("LEAN", "EDGES", "GEN") for r in (8, 16)}, lat
        assert {g["ROWS"] for g in sub.values() if g["last_rows_valid"] < g["ROWS"]} == {8, 16}, lat
        assert any(g["rows_range"] for g in sub.values()), lat
        assert any(CASES[n].get("slot_edges") and g["mode"] == m for n, g in sub.items() for m in (LG.TK_EDGES,
                                                                                                    LG.TK_GEN)), lat
    assert {g["C"] for g in geo.values()} >= {2, 3, 5}
    specs = list(CASES.values())
    assert {s.get("mask") for s in specs} >= {None, "padded", "random"}
    assert any(s["cfg"].get("m_pool_method") == "mean" and not s.get("mask") for s in specs)
    assert any(s["cfg"].get("m_pool_method") == "mean" and s.get("mask") for s in specs)
    for key in ("soft_edges", "norm_coors", "coor_weights_clamp_value", "fourier_features"):
        assert any(key in s["cfg"] for s in specs), key
    # holes: a -1 on the last slot of a group, a whole middle group of -1, an empty row, a self edge
    for name in ("w65_gen8_c5", "w127_edges16", "wb_127_edges16"):
        nbr = build(name)["inputs"]["neighbors"]
        i = np.arange(nbr.shape[1])[None, :, None]
        assert (nbr[:, :, 31] < 0).any() and (nbr[:, :, 63] < 0).any()
        assert (nbr[:, :, 32:64] < 0).all(-1).any() and (nbr < 0).all(-1).any() and (nbr == i).any(), name
    c4 = geometry(CASES["w96_c4"])
    assert (c4["dim"], c4["edge_dim"], c4["B"], c4["N"], c4["k"]) == (256, 4, 2, 4096, 96)


def _holes(nbr, rs, distinct):
    """-1 slots: 20 % at random, the last slot of every group on a third of the rows, slots 32..63 (a whole group, in the
    middle of rows longer than 64) on rows 1 mod 5, every slot on rows 2 mod 7; rows 3 mod 5 hold their own node in
    slot 0 (`distinct`: swapped there, so a row never lists a node twice)."""
    B, N, k = nbr.shape
    nbr[rs.uniform(size=nbr.shape) < 0.2] = -1
    nbr[:, ::3, 31::32] = -1
    nbr[:, 1::5, 32:64] = -1
    nbr[:, 2::7, :] = -1
    for i in range(3, N, 5):
        for b in range(B):
            row = nbr[b, i]
            hit = np.nonzero(row == i)[0]
            if distinct and hit.size:
                row[hit[0]] = row[0]
            row[0] = i
    return nbr


_BUILT = {}


def build(name):
    """The case with bf16 parameters / features / edges, fp32 coordinates and its caller lists."""
    if name in _BUILT:
        return _BUILT[name]
    spec = CASES[name]
    lat = TB.lattice_kind(spec)
    slot = bool(spec.get("slot_edges"))
    case = cases.build_case(dict({k: v for k, v in spec.items() if k not in ("check", "rows", "box", "cell", "k")},
                                 init="xavier", dense_edges=not slot))
    ins = case["inputs"]
    if lat:
        case[lat], ins["coors"] = TB.lattice_inputs(spec, np.random.RandomState(spec["seed"] + 11))
    case["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in case["params"].items()}
    ins["feats"] = util.rounded(ins["feats"], torch.bfloat16)
    ins["coors"] = np.asarray(ins["coors"], np.float32).astype(np.float64)
    if ins.get("edges") is not None:
        ins["edges"] = util.rounded(ins["edges"], torch.bfloat16)
    B, N, k = spec["B"], spec["N"], spec["k"]
    rs = np.random.RandomState(spec["seed"] + 7)
    if slot:     # distinct neighbours per row: the oracle takes per-slot edges as a dense [B, N, N, e] tensor
        nbr = np.stack([np.stack([rs.permutation(N)[:k] for _ in range(N)]) for _ in range(B)])
    else:
        nbr = rs.randint(0, N, (B, N, k))
    ins["neighbors"] = _holes(nbr, rs, slot) if spec.get("holes") else nbr
    if slot:
        ins["edges"] = util.rounded(rs.standard_normal((B, N, k, case["cfg"]["edge_dim"])), torch.bfloat16)
    _BUILT[name] = case
    return case


def windows(name):
    spec = CASES[name]
    return spec.get("check") or [spec.get("rows") or (0, spec["N"])]


def lattice_kw(name):
    case = build(name)
    return {k: case[k] for k in ("box", "cell") if k in case}


def reference(name, rounding=True):
    case = build(name)
    ins = case["inputs"]
    return [(w,) + T.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], edges=ins.get("edges"),
                                      mask=ins.get("mask"), neighbors=ins["neighbors"],
                                      slot_edges=bool(CASES[name].get("slot_edges")), rows=w, rounding=rounding,
                                      **lattice_kw(name))
            for w in windows(name)]


def oracle(name):
    """The fp64 oracle over the same windows: the edge-list oracle, or under a lattice (or for per-slot edges at c4's
    size, where a dense edge tensor would take 1 GB) the float64 restatement torch_reference.layer."""
    case = build(name)
    ins = case["inputs"]
    spec = CASES[name]
    slot = spec.get("slot_edges")
    lat = lattice_kw(name)
    if lat or spec["N"] > 1000:
        with TB.TRI._cell_geometry() if "cell" in lat else contextlib.nullcontext():
            out = []
            for w in windows(name):
                f, x = R.layer(case["params"], case["cfg"], ins["feats"], ins["coors"], None if slot else ins.get("edges"),
                               ins.get("mask"), None, next(iter(lat.values()), None), ins["neighbors"],
                               ins.get("edges") if slot else None, rows=w)
                out.append((w, f.numpy(), x.numpy()))
            return out
    e = ins.get("edges")
    if slot:
        B, N, k = ins["neighbors"].shape
        dense = np.zeros((B, N, N, e.shape[-1]))
        b_, i_, s_ = np.nonzero(ins["neighbors"] >= 0)
        dense[b_, i_, ins["neighbors"][b_, i_, s_]] = e[b_, i_, s_]
        e = dense
    f, x = O.egnn_layer_forward_edge_list(case["params"], case["cfg"], ins["feats"], ins["coors"], ins["neighbors"],
                                          edges=e, mask=ins.get("mask"))
    return [(w, f[:, w[0]:w[1]], x[:, w[0]:w[1]]) for w in windows(name)]


def gates(ref, x_in, outs):
    """test_gpu_tc_boundaries.gates over [(window, feats, coors)] of the reference and [(feats, coors)] outputs."""
    fu, cr, ce, cu = [], [], [], []
    for (w, rf, rx), (gf, gx) in zip(ref, outs):
        floor = 1e-2 * np.abs(rf).max()
        ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(rf), floor))) - 7)
        fu.append((np.abs(gf - rf) / ulp).ravel())
        upd = rx - x_in[:, w[0]:w[1]]
        err = np.abs(gx - rx).max(-1)
        row_upd = np.abs(upd).max(-1)
        cr.append((err / np.maximum(row_upd, 1e-3 * np.abs(upd).max() + 1e-30)).ravel())
        ce.append((gx - rx).ravel())
        cu.append(upd.ravel())
    fu, cr, ce, cu = (np.concatenate(a) for a in (fu, cr, ce, cu))
    return dict(f_ulp_max=float(fu.max()), f_ulp_mean=float(fu.mean()), c_row=float(cr.max()),
                c_rms=float(np.sqrt((ce ** 2).mean() / max((cu ** 2).mean(), 1e-300))))


def oracle_gate(name, oracle_out, x_in, f, x):
    for w, of, ox in oracle_out:
        gf = f[:, w[0]:w[1]].double().cpu().numpy()
        gx = x[:, w[0]:w[1]].double().cpu().numpy()
        assert np.abs(gf - of).max() <= 1e-2 * max(1e-3, np.abs(of).max()), name
        assert np.abs(gx - ox).max() <= 1e-2 * max(np.abs(ox - x_in[:, w[0]:w[1]]).max(), 1.0), name


# ------------------------------------------------------------------ the reference pinned to the oracle (CPU)


@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_unrounded_reference_equals_the_edge_list_oracle_at_k_above_32(masked, mean):
    """Lists of 70 slots (3 groups) with the hole patterns of the table and per-slot edges."""
    spec = dict(kind=L, cfg=dict(dim=16, edge_dim=2, fourier_features=1, soft_edges=True, norm_coors=True,
                                 coor_weights_clamp_value=0.8, m_pool_method="mean" if mean else "sum"),
                B=2, N=90, seed=840, init="xavier", mask="random" if masked else "none")
    c = cases.build_case(spec)
    ins = c["inputs"]
    rs = np.random.RandomState(6)
    k = 70
    nbr = _holes(np.stack([np.stack([rs.permutation(90)[:k] for _ in range(90)]) for _ in range(2)]), rs, True)
    slot = rs.standard_normal((2, 90, k, 2))
    dense = np.zeros((2, 90, 90, 2))
    b_, i_, s_ = np.nonzero(nbr >= 0)
    dense[b_, i_, nbr[b_, i_, s_]] = slot[b_, i_, s_]
    want = O.egnn_layer_forward_edge_list(c["params"], c["cfg"], ins["feats"], ins["coors"], nbr, edges=dense,
                                          mask=ins.get("mask"))
    for edges, per_slot in ((dense, False), (slot, True)):
        got = T.tc_layer_forward(c["params"], c["cfg"], ins["feats"], ins["coors"], edges=edges, mask=ins.get("mask"),
                                 neighbors=nbr, slot_edges=per_slot, rounding=False)
        for g, w in zip(got, want):
            assert np.abs(g - w).max() <= 1e-12 * max(1.0, np.abs(w).max())


# ------------------------------------------------------------------ the GPU runs


def run_gpu(name, rows="spec", lattice=None, dense_edges=False):
    """Forward of the case on the bf16 path.  `dense_edges`: per-slot edges scattered into a dense [B, N, N, e]
    tensor and passed as `edges` instead of `neighbor_edges`."""
    case = build(name)
    spec = CASES[name]
    ins = case["inputs"]
    rows = spec.get("rows") if rows == "spec" else rows
    mod = util.make_module(case, torch.bfloat16)
    dev = "cuda"
    tb = lambda a: None if a is None else torch.from_numpy(np.asarray(a, np.float64)).to(dev, torch.bfloat16)
    lat = {k: torch.as_tensor(np.asarray(v), dtype=torch.float32, device=dev)
           for k, v in (lattice_kw(name) if lattice is None else lattice).items()}
    nbr = torch.from_numpy(ins["neighbors"]).to(dev)
    kw = dict(mask=None if ins.get("mask") is None else torch.from_numpy(ins["mask"]).to(dev), _rows=rows,
              neighbors=nbr, **lat)
    edges = tb(ins.get("edges"))
    if spec.get("slot_edges"):
        if dense_edges:
            B, N, k, e = edges.shape
            dense = torch.zeros(B, N, N, e, dtype=edges.dtype, device=dev)
            b_, i_, s_ = torch.nonzero(nbr >= 0, as_tuple=True)
            dense[b_, i_, nbr[b_, i_, s_].long()] = edges[b_, i_, s_]
            edges = dense
        else:
            kw["neighbor_edges"], edges = edges, None
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("error")
        f, x = mod(tb(ins["feats"]), torch.from_numpy(ins["coors"]).float().to(dev), edges, **kw)
    assert mod.last_path == "bf16-tc", name
    return f, x


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_matches_rounding_matched_reference(name):
    f, x = run_gpu(name)
    assert np.isfinite(f.float().cpu().numpy()).all() and np.isfinite(x.cpu().numpy()).all()
    x_in = build(name)["inputs"]["coors"]
    m = gates(reference(name), x_in, [(f[:, w[0]:w[1]].double().cpu().numpy(), x[:, w[0]:w[1]].double().cpu().numpy())
                                      for w in windows(name)])
    g = geometry(CASES[name], torch.cuda.get_device_properties(0).multi_processor_count)
    print(f"TCW {name} {g['kernel']} k={g['k']} groups={g['groups']} Hp={g['Hp']} "
          + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
    bad = {k: v for k, v in m.items() if not v <= TOL[k]}
    assert not bad, (name, bad)
    oracle_gate(name, oracle(name), x_in, f, x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w96_lean16_clamp", "w128_gen16_rows", "wb_127_edges16", "wc_33_lean8"])
def test_row_range_is_bit_identical_to_the_full_forward(name):
    n = CASES[name]["N"]
    f_full, x_full = run_gpu(name, rows=None)
    for r0, r1 in [(5, n - 3), (37, 38)]:
        f, x = run_gpu(name, rows=(r0, r1))
        assert torch.equal(f[:, r0:r1], f_full[:, r0:r1]) and torch.equal(x[:, r0:r1], x_full[:, r0:r1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w63_edges8_slot", "w128_gen16_rows", "wc_63_edges8_slot"])
def test_per_slot_edges_equal_the_dense_tensor_bit_for_bit(name):
    f_slot, x_slot = run_gpu(name)
    f_dense, x_dense = run_gpu(name, dense_edges=True)
    assert torch.equal(f_slot, f_dense) and torch.equal(x_slot, x_dense)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wb_33_lean8", "wb_127_edges16", "wb_128_gen16_rows"])
def test_a_diagonal_cell_is_the_box_bit_for_bit(name):
    box = np.asarray(lattice_kw(name)["box"])
    cell = np.stack([np.diag(b) for b in box]) if box.ndim == 2 else np.diag(box)
    f_box, x_box = run_gpu(name)
    f_cell, x_cell = run_gpu(name, lattice=dict(cell=cell))
    assert torch.equal(f_box, f_cell) and torch.equal(x_box, x_cell)


# ------------------------------------------------------------------ lists from the layer's own select


SELECT = ["plain", "box", "cell"]
SEL_N, SEL_K, SEL_R, SEL_L = 300, 64, 1.0, [3.0, 3.25, 3.5]


def select_lists(x, mask, k, radius, lat):
    """The all-pairs select (egnn_pytorch.py:237-260) on the pair vectors the kernels form: ranks |x_i - x_j|^2 of
    the (wrapped) pair vector, masked pairs at 1e5, the k smallest; ok = rank <= radius.  Asserts that no selection
    or radius decision lies within 1e-5 (relative) of a tie, so fp32 rounding in the kernel cannot change it."""
    B, N, C = x.shape
    rel = torch.as_tensor(x)[:, :, None, :] - torch.as_tensor(x)[:, None, :, :]
    if lat:
        kind, v = next(iter(lat.items()))
        rel = T.fp32(rel)
        rel = torch.stack([(T.wrap_box if kind == "box" else T.wrap_cell)(rel[b], np.asarray(v), True)
                           for b in range(B)])
    rank = (rel ** 2).sum(-1).numpy()
    pm = mask[:, :, None] & mask[:, None, :]
    rank = np.where(pm, rank, 1e5)
    order = np.argsort(rank, -1, kind="stable")
    vals = np.take_along_axis(rank, order, -1)
    live = vals[..., k - 1] < 1e5
    gap = (vals[..., k] - vals[..., k - 1]) / np.maximum(vals[..., k - 1], 1e-6)
    assert (gap[live] > 1e-5).all(), "a k-th neighbour within rounding of the next one: pick another seed"
    near = np.abs(vals[..., :k] - radius) / radius
    assert (near > 1e-5).all(), "a distance within rounding of valid_radius: pick another seed"
    return order[..., :k], vals[..., :k] <= radius


@pytest.mark.gpu
@pytest.mark.parametrize("kind", SELECT)
def test_own_select_at_k_64_with_valid_radius_and_a_mask(kind):
    spec = dict(kind=L, cfg=dict(dim=64, num_nearest_neighbors=SEL_K, valid_radius=SEL_R, soft_edges=True), B=2,
                N=SEL_N, seed=850 + len(kind), mask="padded")
    case = cases.build_case(dict(spec, init="xavier"))
    ins = case["inputs"]
    rs = np.random.RandomState(spec["seed"] + 3)
    # uniform in the lattice's cell (no ties between distances), moved by whole lattice vectors so that pairs wrap
    A = {"plain": np.diag(SEL_L), "box": np.diag(SEL_L), "cell": TB._grid_cell(rs, SEL_L, 0.5)}[kind]
    frac = rs.uniform(0, 1, (2, SEL_N, 3)) + (rs.randint(-1, 2, (2, SEL_N, 3)) if kind != "plain" else 0)
    ins["coors"] = util.rounded(frac @ A, torch.float32)
    lat = {"plain": {}, "box": {"box": np.asarray(SEL_L)}, "cell": {"cell": util.rounded(A, torch.float32)}}[kind]
    case["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in case["params"].items()}
    ins["feats"] = util.rounded(ins["feats"], torch.bfloat16)
    nbr, ok = select_lists(ins["coors"], ins["mask"], SEL_K, SEL_R, lat)
    assert ok.mean() > 0.2 and (~ok).mean() > 0.2, ok.mean()            # the radius cuts inside the lists
    mod = util.make_module(case, torch.bfloat16)
    dev = "cuda"
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("error")
        f, x = mod(torch.from_numpy(ins["feats"]).to(dev, torch.bfloat16), torch.from_numpy(ins["coors"]).float().to(dev),
                   mask=torch.from_numpy(ins["mask"]).to(dev),
                   **{k: torch.as_tensor(np.asarray(v), dtype=torch.float32, device=dev) for k, v in lat.items()})
    assert mod.last_path == "bf16-tc"
    rf, rx = T.tc_layer_forward(case["params"], case["cfg"], ins["feats"], ins["coors"], mask=ins["mask"],
                                neighbors=nbr, nbr_ok=ok, **lat)
    m = gates([((0, SEL_N), rf, rx)], ins["coors"], [(f.double().cpu().numpy(), x.double().cpu().numpy())])
    print(f"TCW select_{kind} " + " ".join(f"{k}={v:.3e}" for k, v in m.items()))
    assert all(m[k] <= TOL[k] for k in m), m


@pytest.mark.gpu
def test_only_sparse_network_with_expanded_adjacency_above_32():
    """EGNN_Network with only_sparse_neighbors and num_adj_degrees = 2 over a random adjacency: the expanded rows hold
    more than 32 nodes, so k (the largest row sum) is above 32; degree labels make the layer generic."""
    spec = dict(kind=NW, cfg=dict(depth=1, dim=32, only_sparse_neighbors=True, num_adj_degrees=2, adj_dim=2,
                                  soft_edges=True), B=2, N=120, seed=860, adj="random3d", adj_p=0.04, mask="padded",
                init="xavier")
    case = cases.build_case(spec)
    ins = case["inputs"]
    case["params"] = {k: util.rounded(v, torch.bfloat16) for k, v in case["params"].items()}
    ins["coors"] = util.rounded(ins["coors"], torch.float32)
    adj, _ = O.adjacency_degrees(ins["adj_mat"], 2, 2)
    k = int(np.asarray(adj).sum(-1).max())
    assert 32 < k < 120, k
    mod = util.make_module(case, torch.bfloat16)
    dev = "cuda"
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("error")
        f, x = mod(torch.from_numpy(util.rounded(ins["feats"], torch.bfloat16)).to(dev, torch.bfloat16),
                   torch.from_numpy(ins["coors"]).float().to(dev), adj_mat=torch.from_numpy(ins["adj_mat"]).to(dev), mask=torch.from_numpy(ins["mask"]).to(dev))
    assert all(l[1].last_path == "bf16-tc" for l in mod.layers)
    rf, rx = T.tc_network_forward(case["params"], case["ncfg"], util.rounded(ins["feats"], torch.bfloat16), ins["coors"], ins["adj_mat"],
                                  mask=ins["mask"])
    m = gates([((0, 120), rf, rx)], ins["coors"], [(f.double().cpu().numpy(), x.double().cpu().numpy())])
    print("TCW net_sparse_k%d " % k + " ".join(f"{n}={v:.3e}" for n, v in m.items()))
    assert all(m[n] <= TOL[n] for n in m), m
